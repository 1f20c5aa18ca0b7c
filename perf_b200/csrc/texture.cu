// texture.cu -- texture atlas of a triangle mesh: one right-isosceles chart per face, two faces per power-of-two cell, the
// cells packed along the Z-order (Morton) curve of a T x T texture.  Three passes, the caller (ops.texture_atlas) doing the
// density search, the sort and the scans in between: legs (per face, the leg of the right isosceles triangle of the face's
// area), layout (per face, in packing order: UVs and cell record) and texels (per texel of a Morton range: the face it shows
// and the surface point it samples).  Every fp32 operation is an explicit round-to-nearest intrinsic and the chart geometry
// is integer, so the device build and the host build of tests/texture_harness.py (-DPERF_HOST_HARNESS, where each entry
// point runs its body over host arrays in a serial loop) agree bit for bit.
// Rules: perfb200.h (perf_atlas_*); restated in numpy in tests/texture_oracle.py.
#include "common.cuh"

#ifdef __CUDA_ARCH__
#define PERF_FSQRT_RN(a) __fsqrt_rn(a)
#else
#define PERF_FSQRT_RN(a) sqrtf(a)
#endif

namespace perf {

constexpr int ATLAS_MAX_CLASSES = 16;
constexpr int ATLAS_INSET = 3;          // chart leg = cell side - 3 (perfb200.h: the bleed invariant)

struct AtlasClass { int32_t pos0, count, cell0, off0, side; };

enum { ATLAS_LEGS, ATLAS_LAYOUT, ATLAS_TEXELS };

struct AtlasArgs {
    const float* pos; int64_t V;                    // [V,3]
    const int32_t* faces; int64_t F;                // [F,3]
    float* legs;                                    // [F]
    int32_t size;                                   // T
    const int32_t* order;                           // [F] faces in packing order
    AtlasClass cls[ATLAS_MAX_CLASSES]; int n_cls;
    float* uv;                                      // [F,3,2]
    int32_t* rec;                                   // [F,4] offset, side, half, right-angle corner
    int32_t* cells;                                 // [C,4] offset, side, first face, second face (-1: none)
    int64_t C;
    int64_t m0;
    int32_t* tface; float* tpoint;                  // [n], [n,3]
};

__host__ __device__ __forceinline__ void atlas_vertex(const AtlasArgs& a, int32_t v, float (&p)[3])
{
    p[0] = a.pos[3 * (int64_t)v]; p[1] = a.pos[3 * (int64_t)v + 1]; p[2] = a.pos[3 * (int64_t)v + 2];
}

// Z-order: x in the even bits, y in the odd bits.
__host__ __device__ __forceinline__ uint32_t atlas_compact(uint32_t v)
{
    v &= 0x55555555u;
    v = (v | (v >> 1)) & 0x33333333u;
    v = (v | (v >> 2)) & 0x0F0F0F0Fu;
    v = (v | (v >> 4)) & 0x00FF00FFu;
    v = (v | (v >> 8)) & 0x0000FFFFu;
    return v;
}

// Leg of face f: e1 = p1 - p0, e2 = p2 - p0, n = e1 x e2, nn = (nx nx + ny ny) + nz nz, leg = sqrt(sqrt(nn)) = sqrt(2 area).
__host__ __device__ __forceinline__ void atlas_leg(const AtlasArgs& a, int64_t f)
{
    float p0[3], p1[3], p2[3], e1[3], e2[3];
    atlas_vertex(a, a.faces[3 * f], p0); atlas_vertex(a, a.faces[3 * f + 1], p1); atlas_vertex(a, a.faces[3 * f + 2], p2);
    for (int d = 0; d < 3; ++d) { e1[d] = PERF_FSUB_RN(p1[d], p0[d]); e2[d] = PERF_FSUB_RN(p2[d], p0[d]); }
    const float nx = PERF_FSUB_RN(PERF_FMUL_RN(e1[1], e2[2]), PERF_FMUL_RN(e1[2], e2[1]));
    const float ny = PERF_FSUB_RN(PERF_FMUL_RN(e1[2], e2[0]), PERF_FMUL_RN(e1[0], e2[2]));
    const float nz = PERF_FSUB_RN(PERF_FMUL_RN(e1[0], e2[1]), PERF_FMUL_RN(e1[1], e2[0]));
    const float nn = PERF_FADD_RN(PERF_FADD_RN(PERF_FMUL_RN(nx, nx), PERF_FMUL_RN(ny, ny)), PERF_FMUL_RN(nz, nz));
    a.legs[f] = PERF_FSQRT_RN(PERF_FSQRT_RN(nn));
}

// Right-angle corner of face f: the corner k opposite the longest edge, |p_{k+2} - p_{k+1}|^2 = (dx dx + dy dy) + dz dz;
// the lowest k on a tie.
__host__ __device__ __forceinline__ int atlas_corner(const AtlasArgs& a, int64_t f)
{
    float p[3][3];
    for (int k = 0; k < 3; ++k) atlas_vertex(a, a.faces[3 * f + k], p[k]);
    int best = 0;
    float bl = -1.0f;
    for (int k = 0; k < 3; ++k) {
        const float* u = p[(k + 1) % 3];
        const float* w = p[(k + 2) % 3];
        const float dx = PERF_FSUB_RN(w[0], u[0]), dy = PERF_FSUB_RN(w[1], u[1]), dz = PERF_FSUB_RN(w[2], u[2]);
        const float l = PERF_FADD_RN(PERF_FADD_RN(PERF_FMUL_RN(dx, dx), PERF_FMUL_RN(dy, dy)), PERF_FMUL_RN(dz, dz));
        if (l > bl) { bl = l; best = k; }
    }
    return best;
}

// Face at packing position p: its class, cell and half; UVs and record; its cell's entry.
__host__ __device__ __forceinline__ void atlas_layout(const AtlasArgs& a, int64_t p)
{
    int c = 0;
    while (c + 1 < a.n_cls && p >= a.cls[c + 1].pos0) ++c;
    const AtlasClass k = a.cls[c];
    const int32_t r = (int32_t)(p - k.pos0), s = k.side, L = s - ATLAS_INSET, half = r & 1;
    const int32_t cell = k.cell0 + (r >> 1), off = k.off0 + (r >> 1) * s * s;
    const int32_t f = a.order[p];
    const int k0 = atlas_corner(a, f);
    const int32_t x0 = (int32_t)atlas_compact((uint32_t)off), y0 = (int32_t)atlas_compact((uint32_t)off >> 1);
    // doubled texel coordinates (integers below 2^16, so uv = t2 / 2T is exact).  Half 0: right angle at the cell's lower-left
    // corner + (0.5, 0.5), legs along +x (corner k0 + 1) and +y (corner k0 + 2); half 1: the same rotated 180 degrees about
    // the cell's centre.
    const int32_t cx = half ? 2 * (x0 + s) - 1 : 2 * x0 + 1, cy = half ? 2 * (y0 + s) - 1 : 2 * y0 + 1, l2 = half ? -2 * L : 2 * L;
    const int32_t t2[3][2] = {{cx, cy}, {cx + l2, cy}, {cx, cy + l2}};
    const float T2 = (float)(2 * a.size);
    for (int j = 0; j < 3; ++j) {
        const int kk = (k0 + j) % 3;
        a.uv[6 * (int64_t)f + 2 * kk] = PERF_FDIV_RN((float)t2[j][0], T2);
        a.uv[6 * (int64_t)f + 2 * kk + 1] = PERF_FDIV_RN((float)t2[j][1], T2);
    }
    int32_t* rec = a.rec + 4 * (int64_t)f;
    rec[0] = off; rec[1] = s; rec[2] = half; rec[3] = k0;
    int32_t* ce = a.cells + 4 * (int64_t)cell;
    if (half) { ce[3] = f; return; }
    ce[0] = off; ce[1] = s; ce[2] = f;
    if (r + 1 == k.count) ce[3] = -1;
}

// Point of the chart {a >= 0, b >= 0, a + b <= L} nearest to the integer point (a, b), doubled (x2, y2), and the doubled
// squared distance (2a - x2)^2 + (2b - y2)^2: the interior, else the nearest of the bottom, left and hypotenuse edges
// (strictly nearer wins, in that order; the nearest point of a convex set is unique).
__host__ __device__ __forceinline__ int64_t atlas_nearest(int32_t a, int32_t b, int32_t L, int32_t& x2, int32_t& y2)
{
    if (a >= 0 && b >= 0 && a + b <= L) { x2 = 2 * a; y2 = 2 * b; return 0; }
    const int32_t L2 = 2 * L;
    const int32_t cand[3][2] = {{2 * (a < 0 ? 0 : (a > L ? L : a)), 0},
                                {0, 2 * (b < 0 ? 0 : (b > L ? L : b))},
                                {0, 0}};
    int32_t u2 = a - b + L;
    u2 = u2 < 0 ? 0 : (u2 > L2 ? L2 : u2);
    int64_t best = -1;
    for (int e = 0; e < 3; ++e) {
        const int32_t cx = e == 2 ? u2 : cand[e][0], cy = e == 2 ? L2 - u2 : cand[e][1];
        const int64_t dx = 2 * (int64_t)a - cx, dy = 2 * (int64_t)b - cy;
        const int64_t d = dx * dx + dy * dy;
        if (best < 0 || d < best) { best = d; x2 = cx; y2 = cy; }
    }
    return best;
}

// Texel m = m0 + i: its cell (the last whose offset is <= m), the nearer of the cell's charts (the first face on a tie), the
// chart point nearest to the texel centre and its world point.
__host__ __device__ __forceinline__ void atlas_texel(const AtlasArgs& a, int64_t i)
{
    const int64_t m = a.m0 + i;
    int64_t lo = 0, hi = a.C;                       // cells[lo].offset <= m < cells[hi].offset
    while (hi - lo > 1) {
        const int64_t mid = (lo + hi) >> 1;
        if (a.cells[4 * mid] <= m) lo = mid; else hi = mid;
    }
    const int32_t* ce = a.cells + 4 * lo;
    const int32_t s = a.C ? ce[1] : 0;
    if (a.C == 0 || m >= (int64_t)ce[0] + (int64_t)s * s) {
        a.tface[i] = -1;
        for (int d = 0; d < 3; ++d) a.tpoint[3 * i + d] = 0.0f;
        return;
    }
    const uint32_t local = (uint32_t)(m - ce[0]);
    const int32_t x = (int32_t)atlas_compact(local), y = (int32_t)atlas_compact(local >> 1), L = s - ATLAS_INSET;
    // texel centre (x + 0.5, y + 0.5) in the cell; in a chart's frame (right angle at the origin, legs along +a and +b) it
    // sits at the integer point (x, y) for half 0 and (s - 1 - x, s - 1 - y) for half 1
    int32_t x2, y2;
    int32_t face = ce[2];
    const int64_t d0 = atlas_nearest(x, y, L, x2, y2);
    if (ce[3] >= 0) {
        int32_t bx2, by2;
        const int64_t d1 = atlas_nearest(s - 1 - x, s - 1 - y, L, bx2, by2);
        if (d1 < d0) { face = ce[3]; x2 = bx2; y2 = by2; }
    }
    const int k0 = a.rec[4 * (int64_t)face + 3];
    const float beta = PERF_FDIV_RN((float)x2, (float)(2 * L)), gamma = PERF_FDIV_RN((float)y2, (float)(2 * L));
    float pa[3], pb[3], pc[3];
    atlas_vertex(a, a.faces[3 * (int64_t)face + k0], pa);
    atlas_vertex(a, a.faces[3 * (int64_t)face + (k0 + 1) % 3], pb);
    atlas_vertex(a, a.faces[3 * (int64_t)face + (k0 + 2) % 3], pc);
    a.tface[i] = face;
    for (int d = 0; d < 3; ++d)
        a.tpoint[3 * i + d] = PERF_FADD_RN(PERF_FADD_RN(pa[d], PERF_FMUL_RN(beta, PERF_FSUB_RN(pb[d], pa[d]))),
                                           PERF_FMUL_RN(gamma, PERF_FSUB_RN(pc[d], pa[d])));
}

template <int S>
__host__ __device__ __forceinline__ void atlas_body(const AtlasArgs& a, int64_t i)
{
    if (S == ATLAS_LEGS) atlas_leg(a, i);
    else if (S == ATLAS_LAYOUT) atlas_layout(a, i);
    else atlas_texel(a, i);
}

template <int S>
__global__ void __launch_bounds__(128) atlas_kernel(const AtlasArgs a, int64_t n)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) atlas_body<S>(a, i);
}

// The product library launches the kernel; the test harness build runs the same body over host arrays.
template <int S>
static int atlas_run(const AtlasArgs& a, int64_t n, void* stream)
{
    if (n <= 0) return PERF_OK;
#ifdef PERF_HOST_HARNESS
    (void)stream;
    for (int64_t i = 0; i < n; ++i) atlas_body<S>(a, i);
#else
    atlas_kernel<S><<<(unsigned)((n + 127) / 128), 128, 0, (cudaStream_t)stream>>>(a, n);
    PERF_LAUNCH_CHECK();
#endif
    return PERF_OK;
}

}  // namespace perf

using namespace perf;

static int atlas_fill(AtlasArgs& a, const float* vertices, uint64_t V, const int32_t* faces, uint64_t F)
{
    PERF_CHECK_ARG(V < (1ull << 31) && F < (1ull << 29), "mesh of %llu vertices / %llu faces: needs V < 2^31 and F < 2^29",
                   (unsigned long long)V, (unsigned long long)F);
    PERF_CHECK_ARG(F == 0 || (vertices && faces), "NULL vertices or faces");
    memset(&a, 0, sizeof(a));
    a.pos = vertices; a.V = (int64_t)V; a.faces = faces; a.F = (int64_t)F;
    return PERF_OK;
}

extern "C" {
#pragma GCC visibility push(default)

int perf_atlas_legs(const float* d_vertices, uint64_t V, const int32_t* d_faces, uint64_t F, float* d_legs, void* stream)
{
    AtlasArgs a;
    int rc = atlas_fill(a, d_vertices, V, d_faces, F); if (rc) return rc;
    PERF_CHECK_ARG(F == 0 || d_legs, "NULL legs");
    a.legs = d_legs;
    return atlas_run<ATLAS_LEGS>(a, (int64_t)F, stream);
}

int perf_atlas_layout(const float* d_vertices, uint64_t V, const int32_t* d_faces, uint64_t F, int size, const int32_t* d_order,
                      const int32_t* h_classes, int n_classes, float* d_uv, int32_t* d_face_rec, int32_t* d_cells, void* stream)
{
    AtlasArgs a;
    int rc = atlas_fill(a, d_vertices, V, d_faces, F); if (rc) return rc;
    PERF_CHECK_ARG(size >= 256 && size <= 16384 && (size & (size - 1)) == 0, "texture size %d: needs a power of two in [256, 16384]", size);
    PERF_CHECK_ARG(n_classes >= 0 && n_classes <= ATLAS_MAX_CLASSES && (n_classes == 0 || h_classes), "%d size classes", n_classes);
    PERF_CHECK_ARG(F == 0 || (d_order && d_uv && d_face_rec && d_cells), "NULL pointer");
    a.size = size; a.order = d_order; a.uv = d_uv; a.rec = d_face_rec; a.cells = d_cells; a.n_cls = n_classes;
    int64_t pos = 0, cell = 0, off = 0, prev = 1ll << 30;
    for (int c = 0; c < n_classes; ++c) {
        const int32_t* h = h_classes + 5 * c;
        const int64_t s = h[4];
        PERF_CHECK_ARG(h[0] == pos && h[1] > 0 && h[2] == cell && h[3] == off && s >= 4 && s <= size && (s & (s - 1)) == 0 && s < prev,
                       "size class %d is not the next in descending order", c);
        a.cls[c] = {h[0], h[1], h[2], h[3], h[4]};
        pos += h[1]; cell += (h[1] + 1) / 2; off += (h[1] + 1) / 2 * s * s; prev = s;
    }
    PERF_CHECK_ARG(pos == (int64_t)F && off <= (int64_t)size * size, "size classes hold %lld faces in %lld texels, need %llu faces in %d^2",
                   (long long)pos, (long long)off, (unsigned long long)F, size);
    return atlas_run<ATLAS_LAYOUT>(a, (int64_t)F, stream);
}

int perf_atlas_texels(const float* d_vertices, uint64_t V, const int32_t* d_faces, uint64_t F, const int32_t* d_face_rec,
                      const int32_t* d_cells, uint64_t C, uint64_t m0, uint64_t n, int32_t* d_face, float* d_point, void* stream)
{
    AtlasArgs a;
    int rc = atlas_fill(a, d_vertices, V, d_faces, F); if (rc) return rc;
    PERF_CHECK_ARG(C <= F && m0 + n <= (1ull << 28), "%llu cells, texels [%llu, %llu + %llu)", (unsigned long long)C,
                   (unsigned long long)m0, (unsigned long long)m0, (unsigned long long)n);
    PERF_CHECK_ARG(n == 0 || ((C == 0 || (d_face_rec && d_cells)) && d_face && d_point), "NULL pointer");
    a.rec = (int32_t*)d_face_rec; a.cells = (int32_t*)d_cells; a.C = (int64_t)C; a.m0 = (int64_t)m0; a.tface = d_face; a.tpoint = d_point;
    return atlas_run<ATLAS_TEXELS>(a, (int64_t)n, stream);
}

#pragma GCC visibility pop
}
