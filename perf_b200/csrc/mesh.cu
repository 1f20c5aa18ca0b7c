// mesh.cu -- surface extraction from a density lattice: marching tetrahedra on the Freudenthal (Kuhn) decomposition.
// Every lattice cube splits into the 6 tetrahedra that share its main diagonal 000 -> 111, one per axis permutation
// (a, b, c), with vertices V0 = 000, V1 = e_a, V2 = e_a + e_b, V3 = 111.  The decomposition is the same in every cube, so
// neighbouring cubes cut a shared face along the same diagonal and the surface is watertight by construction; a tet has
// 16 inside/outside cases and none is ambiguous.  Every tet edge Vu -> Vv (u < v) is a positive-direction lattice edge
// starting at the node cube + Vu, so a node owns 7 edges: +x, +y, +z, +xy, +xz, +yz, +xyz (dir e = 0..6).
// Two passes with the scans done by the caller (the occupancy sampler's count / write pattern, occ.cu): count writes per
// node the crossing-edge count and the triangle count of the cube whose minimum corner it is; write places vertex
// (node p, dir e) at voff[p] + popc(mask(p) & ((1 << e) - 1)) and the cube's triangles from foff[p] on.
// Rules: perfb200.h (perf_mesh_count); restated in numpy in tests/mesh_oracle.py.
#include "common.cuh"

namespace perf {

struct MeshArgs {
    const float* sigma;          // [rx, ry, rz], x slowest
    int r[3];
    float thr;
    float amin[3], aext[3];
    uint8_t* vcount; uint8_t* fcount;
    const int32_t* voff; const int32_t* foff;
    float* verts; int32_t* faces;
};

__host__ __device__ __forceinline__ int mesh_popc(uint32_t v)
{
#ifdef __CUDA_ARCH__
    return __popc(v);
#else
    return __builtin_popcount(v);
#endif
}

// Offset code of edge direction e (bit 0: +x, bit 1: +y, bit 2: +z) and its inverse.
__host__ __device__ __forceinline__ int edge_code(int e) { return e < 3 ? 1 << e : (e == 6 ? 7 : 7 - (1 << (5 - e))); }
__host__ __device__ __forceinline__ int code_edge(int c)
{
    const int n = mesh_popc((uint32_t)c);
    if (n == 1) return c == 1 ? 0 : (c == 2 ? 1 : 2);
    if (n == 2) return c == 3 ? 3 : (c == 5 ? 4 : 5);
    return 6;
}

__host__ __device__ __forceinline__ int64_t node_index(const MeshArgs& a, int i, int j, int k) { return ((int64_t)i * a.r[1] + j) * a.r[2] + k; }
__host__ __device__ __forceinline__ bool node_inside(const MeshArgs& a, int i, int j, int k) { return a.sigma[node_index(a, i, j, k)] > a.thr; }

// Bit e: edge (node (i,j,k), dir e) lies in the lattice and exactly one of its ends is inside (sigma > thr).
__host__ __device__ __forceinline__ uint32_t node_mask(const MeshArgs& a, int i, int j, int k)
{
    const bool in0 = node_inside(a, i, j, k);
    uint32_t m = 0;
    for (int e = 0; e < 7; ++e) {
        const int c = edge_code(e), ni = i + (c & 1), nj = j + ((c >> 1) & 1), nk = k + (c >> 2);
        if (ni < a.r[0] && nj < a.r[1] && nk < a.r[2] && node_inside(a, ni, nj, nk) != in0) m |= 1u << e;
    }
    return m;
}

// Axis permutation (a, b, c) of tet t = 0..5: (x,y,z) (x,z,y) (y,x,z) (y,z,x) (z,x,y) (z,y,x); odd permutations (t = 1, 2, 5)
// give a negatively oriented tet (V0, V1, V2, V3).
__host__ __device__ __forceinline__ void tet_codes(int t, int (&v)[4])
{
    const int pa = t >> 1, pb = (t == 0 || t == 5) ? 1 : ((t == 1 || t == 3) ? 2 : 0);
    v[0] = 0; v[1] = 1 << pa; v[2] = v[1] | (1 << pb); v[3] = 7;
}
__host__ __device__ __forceinline__ bool tet_odd(int t) { return t == 1 || t == 2 || t == 5; }

// Triangles of tet case m (bit u: vertex u inside) as pairs of tet vertices (one per triangle corner, the edge the corner
// lies on); returns the count.  For a positively oriented tet and an even permutation (u0, u1, u2, u3) of its vertices,
// triangle (u1, u2, u3) faces away from u0.  So, with the quad split along (a,c)-(b,d):
//   1 inside vertex i, (i, j, k, l) even:        (ij, ik, il)              -- a positive scaling of (j, k, l) about i
//   1 outside vertex o, (o, j, k, l) even:       (oj, ol, ok)              -- faces toward o, i.e. away from the inside
//   2 inside a < b, outside c, d, (a,b,c,d) even: (ac, ad, bd), (ac, bd, bc)
// Every triangle's normal then points from the inside vertices to the outside ones: along -grad sigma of the linear
// interpolant.  (i ^ s, s = 0..3) is the even permutation that starts with i.
__host__ __device__ __forceinline__ int tet_triangles(int m, int (&tri)[2][3][2])
{
    const int n = mesh_popc((uint32_t)m);
    if (n == 1 || n == 3) {
        const int u = n == 1 ? (m == 1 ? 0 : m == 2 ? 1 : m == 4 ? 2 : 3) : ((~m & 15) == 1 ? 0 : (~m & 15) == 2 ? 1 : (~m & 15) == 4 ? 2 : 3);
        const int j = u ^ 1, k = u ^ 2, l = u ^ 3;
        tri[0][0][0] = u; tri[0][0][1] = j;
        tri[0][1][0] = u; tri[0][1][1] = n == 1 ? k : l;
        tri[0][2][0] = u; tri[0][2][1] = n == 1 ? l : k;
        return 1;
    }
    if (n == 2) {
        int q[4], nq = 0, o[2], no = 0;
        for (int u = 0; u < 4; ++u) { if ((m >> u) & 1) q[nq++] = u; else o[no++] = u; }
        const int a = q[0], b = q[1];
        const bool odd = (b - a) == 2;                 // (a, b, c, d) with c < d is odd for {0,2} and {1,3}
        const int c = odd ? o[1] : o[0], d = odd ? o[0] : o[1];
        const int t[2][3][2] = {{{a, c}, {a, d}, {b, d}}, {{a, c}, {b, d}, {b, c}}};
        for (int x = 0; x < 2; ++x) for (int y = 0; y < 3; ++y) { tri[x][y][0] = t[x][y][0]; tri[x][y][1] = t[x][y][1]; }
        return 2;
    }
    return 0;
}

// Inside bits of the 8 corners of the cube at (i,j,k), by offset code.
__host__ __device__ __forceinline__ uint32_t cube_corners(const MeshArgs& a, int i, int j, int k)
{
    uint32_t c = 0;
    for (int v = 0; v < 8; ++v) if (node_inside(a, i + (v & 1), j + ((v >> 1) & 1), k + (v >> 2))) c |= 1u << v;
    return c;
}
__host__ __device__ __forceinline__ int tet_case(uint32_t corners, const int (&v)[4])
{
    int m = 0;
    for (int u = 0; u < 4; ++u) m |= (int)((corners >> v[u]) & 1u) << u;
    return m;
}

// Count pass, node p = (i,j,k): crossing edges it owns (<= 7) and triangles of its cube (<= 12; 0 on the far faces).
__host__ __device__ __forceinline__ void mesh_count_node(const MeshArgs& a, int64_t p)
{
    const int k = (int)(p % a.r[2]), j = (int)((p / a.r[2]) % a.r[1]), i = (int)(p / ((int64_t)a.r[2] * a.r[1]));
    a.vcount[p] = (uint8_t)mesh_popc(node_mask(a, i, j, k));
    int nf = 0;
    if (i < a.r[0] - 1 && j < a.r[1] - 1 && k < a.r[2] - 1) {
        const uint32_t corners = cube_corners(a, i, j, k);
        if (corners != 0u && corners != 0xFFu) {
            for (int t = 0; t < 6; ++t) {
                int v[4]; tet_codes(t, v);
                const int n = mesh_popc((uint32_t)tet_case(corners, v));
                nf += (n == 1 || n == 3) ? 1 : (n == 2 ? 2 : 0);
            }
        }
    }
    a.fcount[p] = (uint8_t)nf;
}

// Write pass, node p: its vertices, then its cube's triangles.  Vertex on edge (node a, dir e), b = a + offset(e):
//   t = (thr - sigma_a) / (sigma_b - sigma_a),  per axis d: xa = i_d / (r_d - 1), and where the edge moves along d
//   x01_d = xa + t * ((i_d + 1) / (r_d - 1) - xa), else x01_d = xa;  world_d = aabb_min_d + x01_d * ext_d
// each operation one correctly rounded fp32 operation in this order (no contraction).
__host__ __device__ __forceinline__ void mesh_write_node(const MeshArgs& a, int64_t p)
{
    const int k = (int)(p % a.r[2]), j = (int)((p / a.r[2]) % a.r[1]), i = (int)(p / ((int64_t)a.r[2] * a.r[1]));
    const uint32_t mask = node_mask(a, i, j, k);
    if (mask != 0u) {
        const float sa = a.sigma[p];
        const int ijk[3] = {i, j, k};
        int32_t vi = a.voff[p];
        for (int e = 0; e < 7; ++e) {
            if (!((mask >> e) & 1u)) continue;
            const int c = edge_code(e);
            const float sb = a.sigma[node_index(a, i + (c & 1), j + ((c >> 1) & 1), k + (c >> 2))];
            const float t = PERF_FDIV_RN(PERF_FSUB_RN(a.thr, sa), PERF_FSUB_RN(sb, sa));
            for (int d = 0; d < 3; ++d) {
                const float den = (float)(a.r[d] - 1);
                const float xa = PERF_FDIV_RN((float)ijk[d], den);
                float x = xa;
                if ((c >> d) & 1) x = PERF_FADD_RN(xa, PERF_FMUL_RN(t, PERF_FSUB_RN(PERF_FDIV_RN((float)(ijk[d] + 1), den), xa)));
                a.verts[3 * (int64_t)vi + d] = PERF_FADD_RN(a.amin[d], PERF_FMUL_RN(x, a.aext[d]));
            }
            ++vi;
        }
    }
    if (i >= a.r[0] - 1 || j >= a.r[1] - 1 || k >= a.r[2] - 1) return;
    const uint32_t corners = cube_corners(a, i, j, k);
    if (corners == 0u || corners == 0xFFu) return;
    uint32_t cm[8];                                   // crossing masks of the cube's corners, as needed
    for (int v = 0; v < 8; ++v) cm[v] = 0xFFFFFFFFu;
    int32_t fi = a.foff[p];
    for (int t = 0; t < 6; ++t) {
        int v[4]; tet_codes(t, v);
        int tri[2][3][2];
        const int nt = tet_triangles(tet_case(corners, v), tri);
        for (int x = 0; x < nt; ++x) {
            int32_t idx[3];
            for (int y = 0; y < 3; ++y) {
                int u = tri[x][y][0], w = tri[x][y][1];
                if (u > w) { const int s = u; u = w; w = s; }
                const int cu = v[u], e = code_edge(v[w] ^ cu);       // V_u is contained in V_w: the edge starts at cube + V_u
                if (cm[cu] == 0xFFFFFFFFu) cm[cu] = node_mask(a, i + (cu & 1), j + ((cu >> 1) & 1), k + (cu >> 2));
                idx[y] = a.voff[node_index(a, i + (cu & 1), j + ((cu >> 1) & 1), k + (cu >> 2))] + mesh_popc(cm[cu] & ((1u << e) - 1u));
            }
            if (tet_odd(t)) { const int32_t s = idx[1]; idx[1] = idx[2]; idx[2] = s; }
            a.faces[3 * (int64_t)fi] = idx[0]; a.faces[3 * (int64_t)fi + 1] = idx[1]; a.faces[3 * (int64_t)fi + 2] = idx[2];
            ++fi;
        }
    }
}

template <bool WRITE>
__global__ void __launch_bounds__(128) mesh_kernel(const MeshArgs a, int64_t n)
{
    const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n) return;
    if (WRITE) mesh_write_node(a, p); else mesh_count_node(a, p);
}

}  // namespace perf

using namespace perf;

static int mesh_fill(MeshArgs& a, const float* sigma, const int* res3, float thr, int64_t& n)
{
    PERF_CHECK_ARG(sigma && res3, "NULL pointer");
    PERF_CHECK_ARG(res3[0] >= 2 && res3[1] >= 2 && res3[2] >= 2, "lattice %d x %d x %d: every axis needs >= 2 nodes", res3[0], res3[1], res3[2]);
    const uint64_t nn = (uint64_t)res3[0] * (uint64_t)res3[1] * (uint64_t)res3[2];
    PERF_CHECK_ARG(nn < (1ull << 31), "lattice %d x %d x %d has >= 2^31 nodes", res3[0], res3[1], res3[2]);
    memset(&a, 0, sizeof(a));
    a.sigma = sigma; a.thr = thr;
    for (int d = 0; d < 3; ++d) a.r[d] = res3[d];
    n = (int64_t)nn;
    return PERF_OK;
}

static int mesh_fill_write(MeshArgs& a, const float* aabb6, const int32_t* voff, const int32_t* foff, float* verts, int32_t* faces)
{
    PERF_CHECK_ARG(aabb6 && voff && foff && verts && faces, "NULL pointer");
    for (int d = 0; d < 3; ++d) { a.amin[d] = aabb6[d]; a.aext[d] = aabb6[3 + d] - aabb6[d]; }
    a.voff = voff; a.foff = foff; a.verts = verts; a.faces = faces;
    return PERF_OK;
}

extern "C" {
#pragma GCC visibility push(default)

int perf_mesh_count(const float* d_sigma, const int* h_res3, float threshold, uint8_t* d_vcount, uint8_t* d_fcount, void* stream)
{
    MeshArgs a; int64_t n = 0;
    int rc = mesh_fill(a, d_sigma, h_res3, threshold, n); if (rc) return rc;
    PERF_CHECK_ARG(d_vcount && d_fcount, "NULL counts");
    a.vcount = d_vcount; a.fcount = d_fcount;
    mesh_kernel<false><<<(unsigned)((n + 127) / 128), 128, 0, (cudaStream_t)stream>>>(a, n);
    PERF_LAUNCH_CHECK();
    return PERF_OK;
}

int perf_mesh_write(const float* d_sigma, const int* h_res3, float threshold, const float* h_aabb6, const int32_t* d_voff, const int32_t* d_foff,
                    float* d_vertices, int32_t* d_faces, void* stream)
{
    MeshArgs a; int64_t n = 0;
    int rc = mesh_fill(a, d_sigma, h_res3, threshold, n); if (rc) return rc;
    rc = mesh_fill_write(a, h_aabb6, d_voff, d_foff, d_vertices, d_faces); if (rc) return rc;
    mesh_kernel<true><<<(unsigned)((n + 127) / 128), 128, 0, (cudaStream_t)stream>>>(a, n);
    PERF_LAUNCH_CHECK();
    return PERF_OK;
}

#ifdef PERF_HOST_HARNESS
/* TEST HARNESS ONLY (never compiled into libperfb200.so): the per-node bodies over HOST arrays.  pass 0 = count, 1 = write. */
int perf_host_mesh(int pass, const float* h_sigma, const int* h_res3, float threshold, const float* h_aabb6, uint8_t* h_vcount, uint8_t* h_fcount,
                   const int32_t* h_voff, const int32_t* h_foff, float* h_vertices, int32_t* h_faces)
{
    MeshArgs a; int64_t n = 0;
    int rc = mesh_fill(a, h_sigma, h_res3, threshold, n); if (rc) return rc;
    if (pass == 0) {
        PERF_CHECK_ARG(h_vcount && h_fcount, "NULL counts");
        a.vcount = h_vcount; a.fcount = h_fcount;
        for (int64_t p = 0; p < n; ++p) mesh_count_node(a, p);
    } else {
        rc = mesh_fill_write(a, h_aabb6, h_voff, h_foff, h_vertices, h_faces); if (rc) return rc;
        for (int64_t p = 0; p < n; ++p) mesh_write_node(a, p);
    }
    return PERF_OK;
}
#endif

#pragma GCC visibility pop
}
