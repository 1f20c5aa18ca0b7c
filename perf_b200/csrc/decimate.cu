// decimate.cu -- quadric-error (Garland-Heckbert) edge collapse of a closed, consistently oriented, edge-manifold triangle
// mesh, in rounds of independent collapses.  A round: per half-edge validity, placement and cost; an independent set by two
// integer atomicMin passes over the vertices; the collapses; compaction.  The caller (ops.decimate) builds the per-round
// vertex -> corner adjacency with a stable sort, does the scans and reads one count per round; the library never allocates.
// Every fp64 operation of the bodies is an explicit round-to-nearest intrinsic (never contracted into an FMA), so the device
// build and the host build of tests/decimate_harness.py (-DPERF_HOST_HARNESS, where each entry point runs its body over
// host arrays in a serial loop) agree bit for bit.
// Rules: perfb200.h (perf_decimate_*); restated in numpy in tests/decimate_oracle.py.
#include "common.cuh"

#ifdef __CUDA_ARCH__
#define PERF_DADD_RN(a, b) __dadd_rn((a), (b))
#define PERF_DSUB_RN(a, b) __dsub_rn((a), (b))
#define PERF_DMUL_RN(a, b) __dmul_rn((a), (b))
#define PERF_DDIV_RN(a, b) __ddiv_rn((a), (b))
#define PERF_DSQRT_RN(a) __dsqrt_rn(a)
#define PERF_D2F_RN(a) __double2float_rn(a)
#else
#define PERF_DADD_RN(a, b) ((a) + (b))
#define PERF_DSUB_RN(a, b) ((a) - (b))
#define PERF_DMUL_RN(a, b) ((a) * (b))
#define PERF_DDIV_RN(a, b) ((a) / (b))
#define PERF_DSQRT_RN(a) sqrt(a)
#define PERF_D2F_RN(a) ((float)(a))
#endif

namespace perf {

constexpr int64_t DEC_NO_KEY = 0x7FFFFFFFFFFFFFFFll;   // no candidate edge (above every key: cost bits < 2^31)
constexpr double DEC_COND = 1e-6;                      // det(A) > DEC_COND * trace(A)^3: the 3x3 system is solved

enum { DEC_CHECK, DEC_QUADRICS, DEC_EDGES, DEC_VMIN2, DEC_SELECT, DEC_COLLAPSE, DEC_COMPACT_F, DEC_COMPACT_V,
       DEC_HOOK, DEC_JUMP, DEC_BOX, DEC_DROP_V, DEC_DROP_F, DEC_CYCLES, DEC_CYCLE_SELECT, DEC_CUT };

struct DecArgs {
    float* pos; double* quad; int64_t V;                  // [V,3] fp32, [V,10] fp64
    int32_t* faces; int64_t F;                            // [F,3]
    const int32_t* adj; const int32_t* adj_off;           // corners 3f + k sorted by vertex (stable), offsets [V + 1]
    int64_t* key; float* place;                           // per half-edge [3F], [3F,3]
    int64_t* vmin; int64_t* vmin2; uint8_t* sel;          // m1 [V], m2 [V], selected [3F]
    const int64_t* edges; int64_t n_edges;                // edge ids to collapse
    uint8_t* valive; uint8_t* falive;                     // [V], [F]
    const int32_t* voff; const int32_t* foff;             // exclusive scans of valive / falive
    float* out_pos; double* out_quad; int32_t* out_faces;
    int32_t* flags;
};

// The topological-noise removal stages: the collapse fields plus their own (a separate kernel, so DecArgs keeps its size).
struct DecCleanArgs : DecArgs {
    int32_t* label; int32_t* box; double min_comp;        // component label [V], box [V,6] int32 images, drop diagonal
    int32_t* third; float max_cut;                        // cycle's third vertex [3F], longest perimeter cut
};

struct D3 { double x, y, z; };

__host__ __device__ __forceinline__ D3 dec_pos(const float* p, int64_t v) { return {(double)p[3 * v], (double)p[3 * v + 1], (double)p[3 * v + 2]}; }
__host__ __device__ __forceinline__ D3 dec_sub(D3 a, D3 b) { return {PERF_DSUB_RN(a.x, b.x), PERF_DSUB_RN(a.y, b.y), PERF_DSUB_RN(a.z, b.z)}; }
__host__ __device__ __forceinline__ double dec_dot(D3 a, D3 b)
{
    return PERF_DADD_RN(PERF_DADD_RN(PERF_DMUL_RN(a.x, b.x), PERF_DMUL_RN(a.y, b.y)), PERF_DMUL_RN(a.z, b.z));
}
// (p1 - p0) x (p2 - p0)
__host__ __device__ __forceinline__ D3 dec_normal(D3 p0, D3 p1, D3 p2)
{
    const D3 a = dec_sub(p1, p0), b = dec_sub(p2, p0);
    return {PERF_DSUB_RN(PERF_DMUL_RN(a.y, b.z), PERF_DMUL_RN(a.z, b.y)), PERF_DSUB_RN(PERF_DMUL_RN(a.z, b.x), PERF_DMUL_RN(a.x, b.z)),
            PERF_DSUB_RN(PERF_DMUL_RN(a.x, b.y), PERF_DMUL_RN(a.y, b.x))};
}
__host__ __device__ __forceinline__ int32_t dec_next(const DecArgs& a, int64_t c) { return a.faces[c - c % 3 + (c % 3 + 1) % 3]; }
__host__ __device__ __forceinline__ int32_t dec_prev(const DecArgs& a, int64_t c) { return a.faces[c - c % 3 + (c % 3 + 2) % 3]; }
__host__ __device__ __forceinline__ int32_t dec_valence(const DecArgs& a, int32_t v) { return a.adj_off[v + 1] - a.adj_off[v]; }

__host__ __device__ __forceinline__ void dec_min(int64_t* p, int64_t v)
{
#ifdef __CUDA_ARCH__
    atomicMin((unsigned long long*)p, (unsigned long long)v);     // keys are >= 0: the unsigned order is the signed one
#else
    if (v < *p) *p = v;
#endif
}

// Area-weighted plane quadric of face f: n = (p1 - p0) x (p2 - p0), e = (n / |n|, -(n / |n|) . p0), q = (|n| / 2) e e^T as the
// 10 entries (00 01 02 03 11 12 13 22 23 33); 0 for a zero-area face.
__host__ __device__ __forceinline__ void dec_face_quadric(const DecArgs& a, int64_t f, double (&q)[10])
{
    const D3 p0 = dec_pos(a.pos, a.faces[3 * f]), p1 = dec_pos(a.pos, a.faces[3 * f + 1]), p2 = dec_pos(a.pos, a.faces[3 * f + 2]);
    const D3 n = dec_normal(p0, p1, p2);
    const double nn = dec_dot(n, n);
    if (!(nn > 0.0)) { for (int i = 0; i < 10; ++i) q[i] = 0.0; return; }
    const double len = PERF_DSQRT_RN(nn);
    const D3 u = {PERF_DDIV_RN(n.x, len), PERF_DDIV_RN(n.y, len), PERF_DDIV_RN(n.z, len)};
    const double e[4] = {u.x, u.y, u.z, -dec_dot(u, p0)};
    const double w = PERF_DMUL_RN(0.5, len);
    int t = 0;
    for (int i = 0; i < 4; ++i)
        for (int j = i; j < 4; ++j) q[t++] = PERF_DMUL_RN(w, PERF_DMUL_RN(e[i], e[j]));
}

// Quadric error of the homogeneous point (p, 1): r_i = ((q_i0 x + q_i1 y) + q_i2 z) + q_i3, err = ((r0 x + r1 y) + r2 z) + r3.
__host__ __device__ __forceinline__ double dec_err(const double (&q)[10], D3 p)
{
    const double r0 = PERF_DADD_RN(PERF_DADD_RN(PERF_DADD_RN(PERF_DMUL_RN(q[0], p.x), PERF_DMUL_RN(q[1], p.y)), PERF_DMUL_RN(q[2], p.z)), q[3]);
    const double r1 = PERF_DADD_RN(PERF_DADD_RN(PERF_DADD_RN(PERF_DMUL_RN(q[1], p.x), PERF_DMUL_RN(q[4], p.y)), PERF_DMUL_RN(q[5], p.z)), q[6]);
    const double r2 = PERF_DADD_RN(PERF_DADD_RN(PERF_DADD_RN(PERF_DMUL_RN(q[2], p.x), PERF_DMUL_RN(q[5], p.y)), PERF_DMUL_RN(q[7], p.z)), q[8]);
    const double r3 = PERF_DADD_RN(PERF_DADD_RN(PERF_DADD_RN(PERF_DMUL_RN(q[3], p.x), PERF_DMUL_RN(q[6], p.y)), PERF_DMUL_RN(q[8], p.z)), q[9]);
    return PERF_DADD_RN(PERF_DADD_RN(PERF_DADD_RN(PERF_DMUL_RN(r0, p.x), PERF_DMUL_RN(r1, p.y)), PERF_DMUL_RN(r2, p.z)), r3);
}

__host__ __device__ __forceinline__ D3 dec_round(D3 p, float (&out)[3])
{
    out[0] = PERF_D2F_RN(p.x); out[1] = PERF_D2F_RN(p.y); out[2] = PERF_D2F_RN(p.z);
    return {(double)out[0], (double)out[1], (double)out[2]};
}

// Placement of the collapse of edge (u, w) under q = Q_u + Q_w (perfb200.h states the rule); returns the fp32 cost.
__host__ __device__ __forceinline__ float dec_place(const double (&q)[10], D3 pu, D3 pw, float (&out)[3])
{
    const double a = q[0], b = q[1], c = q[2], d = q[4], e = q[5], f = q[7];
    const double c00 = PERF_DSUB_RN(PERF_DMUL_RN(d, f), PERF_DMUL_RN(e, e)), c01 = PERF_DSUB_RN(PERF_DMUL_RN(c, e), PERF_DMUL_RN(b, f));
    const double c02 = PERF_DSUB_RN(PERF_DMUL_RN(b, e), PERF_DMUL_RN(c, d)), c11 = PERF_DSUB_RN(PERF_DMUL_RN(a, f), PERF_DMUL_RN(c, c));
    const double c12 = PERF_DSUB_RN(PERF_DMUL_RN(b, c), PERF_DMUL_RN(a, e)), c22 = PERF_DSUB_RN(PERF_DMUL_RN(a, d), PERF_DMUL_RN(b, b));
    const double det = PERF_DADD_RN(PERF_DADD_RN(PERF_DMUL_RN(a, c00), PERF_DMUL_RN(b, c01)), PERF_DMUL_RN(c, c02));
    const double tr = PERF_DADD_RN(PERF_DADD_RN(a, d), f);
    const D3 mid = {PERF_DMUL_RN(0.5, PERF_DADD_RN(pu.x, pw.x)), PERF_DMUL_RN(0.5, PERF_DADD_RN(pu.y, pw.y)), PERF_DMUL_RN(0.5, PERF_DADD_RN(pu.z, pw.z))};
    double err;
    bool solved = false;
    if (det > PERF_DMUL_RN(DEC_COND, PERF_DMUL_RN(PERF_DMUL_RN(tr, tr), tr))) {
        const double bx = q[3], by = q[6], bz = q[8];
        const D3 s = {-PERF_DDIV_RN(PERF_DADD_RN(PERF_DADD_RN(PERF_DMUL_RN(c00, bx), PERF_DMUL_RN(c01, by)), PERF_DMUL_RN(c02, bz)), det),
                      -PERF_DDIV_RN(PERF_DADD_RN(PERF_DADD_RN(PERF_DMUL_RN(c01, bx), PERF_DMUL_RN(c11, by)), PERF_DMUL_RN(c12, bz)), det),
                      -PERF_DDIV_RN(PERF_DADD_RN(PERF_DADD_RN(PERF_DMUL_RN(c02, bx), PERF_DMUL_RN(c12, by)), PERF_DMUL_RN(c22, bz)), det)};
        float s32[3];
        const D3 sr = dec_round(s, s32);
        const D3 dm = dec_sub(sr, mid), duw = dec_sub(pu, pw);
        if (dec_dot(dm, dm) <= dec_dot(duw, duw)) {
            out[0] = s32[0]; out[1] = s32[1]; out[2] = s32[2];
            err = dec_err(q, sr);
            solved = true;
        }
    }
    if (!solved) {
        float m32[3];
        const D3 mr = dec_round(mid, m32);
        const double eu = dec_err(q, pu), ew = dec_err(q, pw), em = dec_err(q, mr);
        err = eu; out[0] = (float)pu.x; out[1] = (float)pu.y; out[2] = (float)pu.z;
        if (ew < err) { err = ew; out[0] = (float)pw.x; out[1] = (float)pw.y; out[2] = (float)pw.z; }
        if (em < err) { err = em; out[0] = m32[0]; out[1] = m32[1]; out[2] = m32[2]; }
    }
    return err > 0.0 ? PERF_D2F_RN(err) : 0.0f;
}

// Input check, half-edge i = 3f + k from a = faces[i] to b = next: bit 1 a == b, bit 2 a -> b appears more than once,
// bit 4 b -> a does not appear (open).
__host__ __device__ __forceinline__ void dec_check(const DecArgs& a, int64_t i)
{
    const int32_t u = a.faces[i], w = dec_next(a, i);
    int32_t bits = u == w ? 1 : 0, n_uw = 0, n_wu = 0;
    for (int32_t c = a.adj_off[u]; c < a.adj_off[u + 1]; ++c) n_uw += dec_next(a, a.adj[c]) == w;
    for (int32_t c = a.adj_off[w]; c < a.adj_off[w + 1]; ++c) n_wu += dec_next(a, a.adj[c]) == u;
    if (n_uw != 1) bits |= 2;
    if (n_wu == 0) bits |= 4;
    if (bits) {
#ifdef __CUDA_ARCH__
        atomicOr((int*)a.flags, (int)bits);
#else
        *a.flags |= bits;
#endif
    }
}

// Quadric of vertex v: the face quadrics of its corners, summed in ascending face index (the adjacency's stable order).
__host__ __device__ __forceinline__ void dec_quadrics(const DecArgs& a, int64_t v)
{
    double q[10];
    for (int i = 0; i < 10; ++i) q[i] = 0.0;
    for (int32_t c = a.adj_off[v]; c < a.adj_off[v + 1]; ++c) {
        double fq[10];
        dec_face_quadric(a, a.adj[c] / 3, fq);
        for (int i = 0; i < 10; ++i) q[i] = PERF_DADD_RN(q[i], fq[i]);
    }
    for (int i = 0; i < 10; ++i) a.quad[10 * v + i] = q[i];
}

// Half-edge i from u = faces[i] to w = next, u < w (each undirected edge once): validity, placement, cost, key, m1.
__host__ __device__ __forceinline__ void dec_edge(const DecArgs& a, int64_t i)
{
    a.key[i] = DEC_NO_KEY;
    const int32_t u = a.faces[i], w = dec_next(a, i);
    if (!(u < w)) return;
    // link condition |N(u) n N(w)| = 2 and the two opposite vertices: N(v) is the set of next vertices of v's corners
    int32_t o2 = -1, link = 0;
    for (int32_t c = a.adj_off[w]; c < a.adj_off[w + 1]; ++c) if (dec_next(a, a.adj[c]) == u) o2 = dec_prev(a, a.adj[c]);
    for (int32_t c = a.adj_off[u]; c < a.adj_off[u + 1]; ++c) {
        const int32_t x = dec_next(a, a.adj[c]);
        for (int32_t c2 = a.adj_off[w]; c2 < a.adj_off[w + 1]; ++c2)
            if (dec_next(a, a.adj[c2]) == x) { ++link; break; }
    }
    const int32_t o1 = dec_prev(a, i);
    if (link != 2 || o2 < 0 || dec_valence(a, o1) <= 3 || dec_valence(a, o2) <= 3) return;
    double q[10];
    for (int t = 0; t < 10; ++t) q[t] = PERF_DADD_RN(a.quad[10 * (int64_t)u + t], a.quad[10 * (int64_t)w + t]);
    float p32[3];
    const float cost = dec_place(q, dec_pos(a.pos, u), dec_pos(a.pos, w), p32);
    const D3 p = {(double)p32[0], (double)p32[1], (double)p32[2]};
    // no surviving face of star(u) u star(w) flips (zero-area faces exempt)
    for (int side = 0; side < 2; ++side) {
        const int32_t v = side ? w : u, o = side ? u : w;
        for (int32_t c = a.adj_off[v]; c < a.adj_off[v + 1]; ++c) {
            const int64_t g = a.adj[c] / 3;
            const int j = a.adj[c] % 3;
            const int32_t f0 = a.faces[3 * g], f1 = a.faces[3 * g + 1], f2 = a.faces[3 * g + 2];
            if (f0 == o || f1 == o || f2 == o) continue;                    // one of the two faces the collapse removes
            const D3 p0 = dec_pos(a.pos, f0), p1 = dec_pos(a.pos, f1), p2 = dec_pos(a.pos, f2);
            const D3 nb = dec_normal(p0, p1, p2);
            if (dec_dot(nb, nb) == 0.0) continue;
            const D3 na = dec_normal(j == 0 ? p : p0, j == 1 ? p : p1, j == 2 ? p : p2);
            if (!(dec_dot(nb, na) > 0.0)) return;
        }
    }
    uint32_t bits;
    memcpy(&bits, &cost, sizeof(bits));
    const int64_t k = (int64_t)((uint64_t)bits << 32 | (uint64_t)i);
    a.key[i] = k;
    for (int d = 0; d < 3; ++d) a.place[3 * i + d] = p32[d];
    dec_min(&a.vmin[u], k);
    dec_min(&a.vmin[w], k);
}

// m2[u] = min(m1[u], m1 of every neighbour): half-edge u -> w (both directions of every edge exist).
__host__ __device__ __forceinline__ void dec_vmin2(const DecArgs& a, int64_t i) { dec_min(&a.vmin2[a.faces[i]], a.vmin[dec_next(a, i)]); }

__host__ __device__ __forceinline__ void dec_select(const DecArgs& a, int64_t i)
{
    const int64_t k = a.key[i];
    a.sel[i] = k != DEC_NO_KEY && a.vmin2[a.faces[i]] == k && a.vmin2[dec_next(a, i)] == k;
}

// Collapse of selected edge e: w into u at the placement.  The selected edges' stars are disjoint, so no two threads touch
// the same face or vertex.
__host__ __device__ __forceinline__ void dec_collapse(const DecArgs& a, int64_t s)
{
    const int64_t e = a.edges[s];
    const int32_t u = a.faces[e], w = dec_next(a, e);
    for (int t = 0; t < 10; ++t) a.quad[10 * (int64_t)u + t] = PERF_DADD_RN(a.quad[10 * (int64_t)u + t], a.quad[10 * (int64_t)w + t]);
    for (int d = 0; d < 3; ++d) a.pos[3 * (int64_t)u + d] = a.place[3 * e + d];
    a.valive[w] = 0;
    for (int32_t c = a.adj_off[w]; c < a.adj_off[w + 1]; ++c) {
        const int64_t g = a.adj[c] / 3;
        if (a.faces[3 * g] == u || a.faces[3 * g + 1] == u || a.faces[3 * g + 2] == u) a.falive[g] = 0;
        else a.faces[a.adj[c]] = u;
    }
}

__host__ __device__ __forceinline__ void dec_compact_face(const DecArgs& a, int64_t f)
{
    if (!a.falive[f]) return;
    for (int d = 0; d < 3; ++d) a.out_faces[3 * (int64_t)a.foff[f] + d] = a.voff[a.faces[3 * f + d]];
}

__host__ __device__ __forceinline__ void dec_compact_vertex(const DecArgs& a, int64_t v)
{
    if (!a.valive[v]) return;
    const int64_t o = a.voff[v];
    for (int d = 0; d < 3; ++d) a.out_pos[3 * o + d] = a.pos[3 * v + d];
    for (int t = 0; t < 10; ++t) a.out_quad[10 * o + t] = a.quad[10 * v + t];
}

// ---- topological-noise removal: components, their boxes and the drop; short non-face 3-cycles and the cut along them.

__host__ __device__ __forceinline__ void dec_flag(int32_t* p)
{
#ifdef __CUDA_ARCH__
    atomicOr((int*)p, 1);
#else
    *p |= 1;
#endif
}

// Hook, half-edge u -> w: the label of u's label drops to w's when that is smaller (a forest whose parents are smaller).
__host__ __device__ __forceinline__ void dec_hook(const DecCleanArgs& a, int64_t i)
{
    const int32_t lu = a.label[a.faces[i]], lw = a.label[dec_next(a, i)];
    if (!(lw < lu)) return;
#ifdef __CUDA_ARCH__
    atomicMin((int*)&a.label[lu], (int)lw);
#else
    if (lw < a.label[lu]) a.label[lu] = lw;
#endif
    dec_flag(a.flags);
}

// Pointer jump of vertex v to its root.  Other threads only lower labels to ancestors, so any value read is an ancestor.
__host__ __device__ __forceinline__ void dec_jump(const DecCleanArgs& a, int64_t v)
{
    volatile int32_t* lab = a.label;
    int32_t l = lab[v], n;
    while ((n = lab[l]) != l) l = n;
    if (l != lab[v]) { lab[v] = l; dec_flag(a.flags); }
}

// Order-preserving int32 image of an fp32 value (and its inverse: the same map).
__host__ __device__ __forceinline__ int32_t dec_ord(int32_t b) { return b >= 0 ? b : b ^ 0x7FFFFFFF; }

__host__ __device__ __forceinline__ void dec_box(const DecCleanArgs& a, int64_t v)
{
    const int64_t l = a.label[v];
    for (int d = 0; d < 3; ++d) {
        int32_t b;
        memcpy(&b, &a.pos[3 * v + d], sizeof(b));
        b = dec_ord(b);
#ifdef __CUDA_ARCH__
        atomicMin((int*)&a.box[6 * l + d], (int)b);
        atomicMax((int*)&a.box[6 * l + 3 + d], (int)b);
#else
        if (b < a.box[6 * l + d]) a.box[6 * l + d] = b;
        if (b > a.box[6 * l + 3 + d]) a.box[6 * l + 3 + d] = b;
#endif
    }
}

// Vertex v survives iff the diagonal^2 of its component's box, (dx^2 + dy^2) + dz^2 in fp64, is not below min_comp^2.
__host__ __device__ __forceinline__ void dec_drop_vertex(const DecCleanArgs& a, int64_t v)
{
    const int64_t l = a.label[v];
    double e[3];
    for (int d = 0; d < 3; ++d) {
        const int32_t lo = dec_ord(a.box[6 * l + d]), hi = dec_ord(a.box[6 * l + 3 + d]);
        float flo, fhi;
        memcpy(&flo, &lo, sizeof(flo));
        memcpy(&fhi, &hi, sizeof(fhi));
        e[d] = PERF_DSUB_RN((double)fhi, (double)flo);
    }
    const double d2 = PERF_DADD_RN(PERF_DADD_RN(PERF_DMUL_RN(e[0], e[0]), PERF_DMUL_RN(e[1], e[1])), PERF_DMUL_RN(e[2], e[2]));
    a.valive[v] = !(d2 < PERF_DMUL_RN(a.min_comp, a.min_comp));
}

__host__ __device__ __forceinline__ void dec_drop_face(const DecCleanArgs& a, int64_t f) { a.falive[f] = a.valive[a.faces[3 * f]]; }

// Fan step around v from corner c: v's corner whose next is c's prev (-1 if none).
__host__ __device__ __forceinline__ int32_t dec_fan_step(const DecArgs& a, int32_t v, int32_t c)
{
    const int32_t p = dec_prev(a, c);
    for (int32_t t = a.adj_off[v]; t < a.adj_off[v + 1]; ++t) if (dec_next(a, a.adj[t]) == p) return a.adj[t];
    return -1;
}

// v is vertex-manifold iff the fan walk from its first corner visits all its corners before it returns.
__host__ __device__ __forceinline__ bool dec_manifold(const DecArgs& a, int32_t v)
{
    const int32_t n = dec_valence(a, v), c0 = a.adj[a.adj_off[v]];
    int32_t c = c0, k = 0;
    do { c = dec_fan_step(a, v, c); ++k; } while (c >= 0 && c != c0 && k <= n);
    return c == c0 && k == n;
}

__host__ __device__ __forceinline__ double dec_len(D3 p, D3 q) { const D3 d = dec_sub(p, q); return PERF_DSQRT_RN(dec_dot(d, d)); }

// Half-edge i from u to w, u < w, link count > 2: the non-face 3-cycle u -> w -> x (x > w, not an opposite vertex, u w x
// vertex-manifold) of smallest (perimeter, x) with perimeter <= max_cut; key, third vertex, m1 over u, w, x.
__host__ __device__ __forceinline__ void dec_cycles(const DecCleanArgs& a, int64_t i)
{
    a.key[i] = DEC_NO_KEY;
    const int32_t u = a.faces[i], w = dec_next(a, i);
    if (!(u < w)) return;
    int32_t o2 = -1, link = 0;
    for (int32_t c = a.adj_off[w]; c < a.adj_off[w + 1]; ++c) if (dec_next(a, a.adj[c]) == u) o2 = dec_prev(a, a.adj[c]);
    for (int32_t c = a.adj_off[u]; c < a.adj_off[u + 1]; ++c) {
        const int32_t x = dec_next(a, a.adj[c]);
        for (int32_t c2 = a.adj_off[w]; c2 < a.adj_off[w + 1]; ++c2)
            if (dec_next(a, a.adj[c2]) == x) { ++link; break; }
    }
    if (link <= 2 || !dec_manifold(a, u) || !dec_manifold(a, w)) return;
    const int32_t o1 = dec_prev(a, i);
    const D3 pu = dec_pos(a.pos, u), pw = dec_pos(a.pos, w);
    const double luw = dec_len(pu, pw);
    float best = 0.0f;
    int32_t bx = -1;
    for (int32_t c = a.adj_off[u]; c < a.adj_off[u + 1]; ++c) {
        const int32_t x = dec_next(a, a.adj[c]);
        if (x <= w || x == o1 || x == o2) continue;
        bool in_w = false;
        for (int32_t c2 = a.adj_off[w]; c2 < a.adj_off[w + 1]; ++c2) in_w |= dec_next(a, a.adj[c2]) == x;
        if (!in_w) continue;
        const D3 px = dec_pos(a.pos, x);
        const float p = PERF_D2F_RN(PERF_DADD_RN(PERF_DADD_RN(luw, dec_len(pw, px)), dec_len(px, pu)));
        if (!(p <= a.max_cut) || (bx >= 0 && (p > best || (p == best && x > bx))) || !dec_manifold(a, x)) continue;
        best = p; bx = x;
    }
    if (bx < 0) return;
    uint32_t bits;
    memcpy(&bits, &best, sizeof(bits));
    const int64_t k = (int64_t)((uint64_t)bits << 32 | (uint64_t)i);
    a.key[i] = k;
    a.third[i] = bx;
    dec_min(&a.vmin[u], k);
    dec_min(&a.vmin[w], k);
    dec_min(&a.vmin[bx], k);
}

__host__ __device__ __forceinline__ void dec_cycle_select(const DecCleanArgs& a, int64_t i)
{
    const int64_t k = a.key[i];
    a.sel[i] = k != DEC_NO_KEY && a.vmin2[a.faces[i]] == k && a.vmin2[dec_next(a, i)] == k && a.vmin2[a.third[i]] == k;
}

// Cut along selected cycle s (half-edge e = edges[s], u -> w -> x): in each cycle vertex's left arc (from the face of its
// outgoing cycle half-edge, stepping around the fan, to the face of its incoming one) the vertex becomes its copy at
// V + 3s + j; caps (u, w, x) and (u', x', w') at F + 2s.  All three arcs are walked before any corner is rewritten: the face
// of u -> w ends w's arc, and rewriting u there first would hide it.  The arcs' interior spokes are not cycle vertices, so
// the second walk of each arc, by its length, is not disturbed by the other arcs' rewrites.
__host__ __device__ __forceinline__ void dec_cut(const DecCleanArgs& a, int64_t s)
{
    const int64_t e = a.edges[s];
    const int32_t cyc[3] = {a.faces[e], dec_next(a, e), a.third[e]};
    int32_t start[3], len[3];
    for (int j = 0; j < 3; ++j) {
        const int32_t v = cyc[j], n = cyc[(j + 1) % 3], p = cyc[(j + 2) % 3];
        int32_t c = -1;
        for (int32_t t = a.adj_off[v]; t < a.adj_off[v + 1]; ++t) if (dec_next(a, a.adj[t]) == n) c = a.adj[t];
        start[j] = c;
        int32_t k = 1;
        while (dec_prev(a, c) != p) { c = dec_fan_step(a, v, c); ++k; }
        len[j] = k;
    }
    for (int j = 0; j < 3; ++j) {
        const int32_t v = cyc[j], vn = (int32_t)(a.V + 3 * s + j);
        int32_t c = start[j];
        for (int32_t k = 0; k < len[j]; ++k) {
            const int32_t next = k + 1 < len[j] ? dec_fan_step(a, v, c) : -1;
            a.faces[c] = vn;
            c = next;
        }
        for (int d = 0; d < 3; ++d) a.pos[3 * (int64_t)vn + d] = a.pos[3 * (int64_t)v + d];
        for (int t = 0; t < 10; ++t) a.quad[10 * (int64_t)vn + t] = a.quad[10 * (int64_t)v + t];
    }
    int32_t* cap = a.faces + 3 * (a.F + 2 * s);
    const int32_t b = (int32_t)(a.V + 3 * s);
    cap[0] = cyc[0]; cap[1] = cyc[1]; cap[2] = cyc[2];
    cap[3] = b; cap[4] = b + 2; cap[5] = b + 1;
}

template <int S>
__host__ __device__ __forceinline__ void dec_body(const DecArgs& a, int64_t i)
{
    if (S == DEC_CHECK) dec_check(a, i);
    else if (S == DEC_QUADRICS) dec_quadrics(a, i);
    else if (S == DEC_EDGES) dec_edge(a, i);
    else if (S == DEC_VMIN2) dec_vmin2(a, i);
    else if (S == DEC_SELECT) dec_select(a, i);
    else if (S == DEC_COLLAPSE) dec_collapse(a, i);
    else if (S == DEC_COMPACT_F) dec_compact_face(a, i);
    else dec_compact_vertex(a, i);
}

template <int S>
__host__ __device__ __forceinline__ void dec_clean_body(const DecCleanArgs& a, int64_t i)
{
    if (S == DEC_HOOK) dec_hook(a, i);
    else if (S == DEC_JUMP) dec_jump(a, i);
    else if (S == DEC_BOX) dec_box(a, i);
    else if (S == DEC_DROP_V) dec_drop_vertex(a, i);
    else if (S == DEC_DROP_F) dec_drop_face(a, i);
    else if (S == DEC_CYCLES) dec_cycles(a, i);
    else if (S == DEC_CYCLE_SELECT) dec_cycle_select(a, i);
    else dec_cut(a, i);
}

template <int S>
__global__ void __launch_bounds__(128) decimate_kernel(const DecArgs a, int64_t n)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) dec_body<S>(a, i);
}

template <int S>
__global__ void __launch_bounds__(128) decimate_clean_kernel(const DecCleanArgs a, int64_t n)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) dec_clean_body<S>(a, i);
}

// The product library launches the kernel; the test harness build runs the same body over host arrays.
template <int S>
static int dec_run(const DecArgs& a, int64_t n, void* stream)
{
    if (n <= 0) return PERF_OK;
#ifdef PERF_HOST_HARNESS
    (void)stream;
    for (int64_t i = 0; i < n; ++i) dec_body<S>(a, i);
#else
    decimate_kernel<S><<<(unsigned)((n + 127) / 128), 128, 0, (cudaStream_t)stream>>>(a, n);
    PERF_LAUNCH_CHECK();
#endif
    return PERF_OK;
}

template <int S>
static int dec_run(const DecCleanArgs& a, int64_t n, void* stream)
{
    if (n <= 0) return PERF_OK;
#ifdef PERF_HOST_HARNESS
    (void)stream;
    for (int64_t i = 0; i < n; ++i) dec_clean_body<S>(a, i);
#else
    decimate_clean_kernel<S><<<(unsigned)((n + 127) / 128), 128, 0, (cudaStream_t)stream>>>(a, n);
    PERF_LAUNCH_CHECK();
#endif
    return PERF_OK;
}

}  // namespace perf

using namespace perf;

static int dec_fill(DecArgs& a, uint64_t V, const int32_t* faces, uint64_t F, const int32_t* adj, const int32_t* adj_off)
{
    PERF_CHECK_ARG(V < (1ull << 31) && 3 * F < (1ull << 31), "mesh of %llu vertices / %llu faces: needs V < 2^31 and 3F < 2^31",
                   (unsigned long long)V, (unsigned long long)F);
    PERF_CHECK_ARG(F == 0 || (faces && adj && adj_off), "NULL faces or adjacency");
    memset(&a, 0, sizeof(a));
    a.V = (int64_t)V; a.faces = (int32_t*)faces; a.F = (int64_t)F; a.adj = adj; a.adj_off = adj_off;
    return PERF_OK;
}

extern "C" {
#pragma GCC visibility push(default)

int perf_decimate_check(const int32_t* d_faces, uint64_t F, uint64_t V, const int32_t* d_adj, const int32_t* d_adj_off, int32_t* d_flags, void* stream)
{
    DecArgs a;
    int rc = dec_fill(a, V, d_faces, F, d_adj, d_adj_off); if (rc) return rc;
    PERF_CHECK_ARG(d_flags, "NULL flags");
    a.flags = d_flags;
    return dec_run<DEC_CHECK>(a, 3 * (int64_t)F, stream);
}

int perf_decimate_quadrics(const float* d_vertices, uint64_t V, const int32_t* d_faces, uint64_t F, const int32_t* d_adj,
                           const int32_t* d_adj_off, double* d_quadrics, void* stream)
{
    DecArgs a;
    int rc = dec_fill(a, V, d_faces, F, d_adj, d_adj_off); if (rc) return rc;
    PERF_CHECK_ARG(V == 0 || (d_vertices && d_quadrics && d_adj_off), "NULL vertices, quadrics or adjacency");
    a.pos = (float*)d_vertices; a.quad = d_quadrics;
    return dec_run<DEC_QUADRICS>(a, (int64_t)V, stream);
}

int perf_decimate_edges(const float* d_vertices, const double* d_quadrics, uint64_t V, const int32_t* d_faces, uint64_t F,
                        const int32_t* d_adj, const int32_t* d_adj_off, int64_t* d_key, float* d_place, int64_t* d_vmin, void* stream)
{
    DecArgs a;
    int rc = dec_fill(a, V, d_faces, F, d_adj, d_adj_off); if (rc) return rc;
    PERF_CHECK_ARG(F == 0 || (d_vertices && d_quadrics && d_key && d_place && d_vmin), "NULL pointer");
    a.pos = (float*)d_vertices; a.quad = (double*)d_quadrics; a.key = d_key; a.place = d_place; a.vmin = d_vmin;
    return dec_run<DEC_EDGES>(a, 3 * (int64_t)F, stream);
}

int perf_decimate_select(const int32_t* d_faces, uint64_t F, uint64_t V, const int64_t* d_key, const int64_t* d_vmin, int64_t* d_vmin2,
                         uint8_t* d_selected, void* stream)
{
    DecArgs a;
    PERF_CHECK_ARG(V < (1ull << 31) && 3 * F < (1ull << 31), "mesh too large");
    PERF_CHECK_ARG(F == 0 || (d_faces && d_key && d_vmin && d_vmin2 && d_selected), "NULL pointer");
    memset(&a, 0, sizeof(a));
    a.V = (int64_t)V; a.F = (int64_t)F; a.faces = (int32_t*)d_faces;
    a.key = (int64_t*)d_key; a.vmin = (int64_t*)d_vmin; a.vmin2 = d_vmin2; a.sel = d_selected;
    int rc = dec_run<DEC_VMIN2>(a, 3 * (int64_t)F, stream); if (rc) return rc;
    return dec_run<DEC_SELECT>(a, 3 * (int64_t)F, stream);
}

int perf_decimate_collapse(const int64_t* d_edges, uint64_t n, float* d_vertices, double* d_quadrics, uint64_t V, int32_t* d_faces, uint64_t F,
                           const int32_t* d_adj, const int32_t* d_adj_off, const float* d_place, uint8_t* d_valive, uint8_t* d_falive, void* stream)
{
    DecArgs a;
    int rc = dec_fill(a, V, d_faces, F, d_adj, d_adj_off); if (rc) return rc;
    PERF_CHECK_ARG(n <= F / 2, "%llu collapses on %llu faces", (unsigned long long)n, (unsigned long long)F);
    PERF_CHECK_ARG(n == 0 || (d_edges && d_vertices && d_quadrics && d_place && d_valive && d_falive), "NULL pointer");
    a.edges = d_edges; a.n_edges = (int64_t)n; a.pos = d_vertices; a.quad = d_quadrics; a.place = (float*)d_place;
    a.valive = d_valive; a.falive = d_falive;
    return dec_run<DEC_COLLAPSE>(a, (int64_t)n, stream);
}

int perf_decimate_compact(const float* d_vertices, const double* d_quadrics, uint64_t V, const uint8_t* d_valive, const int32_t* d_voff,
                          const int32_t* d_faces, uint64_t F, const uint8_t* d_falive, const int32_t* d_foff,
                          float* d_out_vertices, double* d_out_quadrics, int32_t* d_out_faces, void* stream)
{
    DecArgs a;
    PERF_CHECK_ARG(V < (1ull << 31) && 3 * F < (1ull << 31), "mesh too large");
    PERF_CHECK_ARG(V == 0 || (d_vertices && d_quadrics && d_valive && d_voff && d_out_vertices && d_out_quadrics), "NULL vertex array");
    PERF_CHECK_ARG(F == 0 || (d_faces && d_falive && d_foff && d_out_faces && d_voff), "NULL face array");
    memset(&a, 0, sizeof(a));
    a.pos = (float*)d_vertices; a.quad = (double*)d_quadrics; a.V = (int64_t)V; a.valive = (uint8_t*)d_valive; a.voff = d_voff;
    a.faces = (int32_t*)d_faces; a.F = (int64_t)F; a.falive = (uint8_t*)d_falive; a.foff = d_foff;
    a.out_pos = d_out_vertices; a.out_quad = d_out_quadrics; a.out_faces = d_out_faces;
    int rc = dec_run<DEC_COMPACT_F>(a, (int64_t)F, stream); if (rc) return rc;
    return dec_run<DEC_COMPACT_V>(a, (int64_t)V, stream);
}

int perf_decimate_components(const int32_t* d_faces, uint64_t F, uint64_t V, int32_t* d_label, int32_t* d_changed, void* stream)
{
    DecCleanArgs a;
    PERF_CHECK_ARG(V < (1ull << 31) && 3 * F < (1ull << 31), "mesh too large");
    PERF_CHECK_ARG(V == 0 || (d_label && d_changed && (F == 0 || d_faces)), "NULL pointer");
    memset(&a, 0, sizeof(a));
    a.V = (int64_t)V; a.F = (int64_t)F; a.faces = (int32_t*)d_faces; a.label = d_label; a.flags = d_changed;
    int rc = dec_run<DEC_HOOK>(a, 3 * (int64_t)F, stream); if (rc) return rc;
    return dec_run<DEC_JUMP>(a, (int64_t)V, stream);
}

int perf_decimate_component_box(const float* d_vertices, uint64_t V, const int32_t* d_faces, uint64_t F, const int32_t* d_label,
                                double min_component, int32_t* d_box, uint8_t* d_valive, uint8_t* d_falive, void* stream)
{
    DecCleanArgs a;
    PERF_CHECK_ARG(V < (1ull << 31) && 3 * F < (1ull << 31), "mesh too large");
    PERF_CHECK_ARG(V == 0 || (d_vertices && d_label && d_box && d_valive), "NULL vertex array");
    PERF_CHECK_ARG(F == 0 || (d_faces && d_falive), "NULL face array");
    PERF_CHECK_ARG(min_component >= 0.0, "min_component %g < 0", min_component);
    memset(&a, 0, sizeof(a));
    a.pos = (float*)d_vertices; a.V = (int64_t)V; a.faces = (int32_t*)d_faces; a.F = (int64_t)F; a.label = (int32_t*)d_label;
    a.min_comp = min_component; a.box = d_box; a.valive = d_valive; a.falive = d_falive;
    int rc = dec_run<DEC_BOX>(a, (int64_t)V, stream); if (rc) return rc;
    rc = dec_run<DEC_DROP_V>(a, (int64_t)V, stream); if (rc) return rc;
    return dec_run<DEC_DROP_F>(a, (int64_t)F, stream);
}

int perf_decimate_cycles(const float* d_vertices, uint64_t V, const int32_t* d_faces, uint64_t F, const int32_t* d_adj,
                         const int32_t* d_adj_off, float max_cut, int64_t* d_key, int32_t* d_third, int64_t* d_vmin, void* stream)
{
    DecCleanArgs a;
    memset(&a, 0, sizeof(a));
    int rc = dec_fill(a, V, d_faces, F, d_adj, d_adj_off); if (rc) return rc;
    PERF_CHECK_ARG(F == 0 || (d_vertices && d_key && d_third && d_vmin), "NULL pointer");
    a.pos = (float*)d_vertices; a.max_cut = max_cut; a.key = d_key; a.third = d_third; a.vmin = d_vmin;
    return dec_run<DEC_CYCLES>(a, 3 * (int64_t)F, stream);
}

int perf_decimate_cycle_select(const int32_t* d_faces, uint64_t F, uint64_t V, const int64_t* d_key, const int32_t* d_third,
                               const int64_t* d_vmin, int64_t* d_vmin2, uint8_t* d_selected, void* stream)
{
    DecCleanArgs a;
    PERF_CHECK_ARG(V < (1ull << 31) && 3 * F < (1ull << 31), "mesh too large");
    PERF_CHECK_ARG(F == 0 || (d_faces && d_key && d_third && d_vmin && d_vmin2 && d_selected), "NULL pointer");
    memset(&a, 0, sizeof(a));
    a.V = (int64_t)V; a.F = (int64_t)F; a.faces = (int32_t*)d_faces;
    a.key = (int64_t*)d_key; a.third = (int32_t*)d_third; a.vmin = (int64_t*)d_vmin; a.vmin2 = d_vmin2; a.sel = d_selected;
    int rc = dec_run<DEC_VMIN2>(static_cast<const DecArgs&>(a), 3 * (int64_t)F, stream); if (rc) return rc;
    return dec_run<DEC_CYCLE_SELECT>(a, 3 * (int64_t)F, stream);
}

int perf_decimate_cut(const int64_t* d_cycles, uint64_t n, const int32_t* d_third, float* d_vertices, double* d_quadrics, uint64_t V,
                      int32_t* d_faces, uint64_t F, const int32_t* d_adj, const int32_t* d_adj_off, void* stream)
{
    DecCleanArgs a;
    memset(&a, 0, sizeof(a));
    int rc = dec_fill(a, V, d_faces, F, d_adj, d_adj_off); if (rc) return rc;
    PERF_CHECK_ARG(V + 3 * n < (1ull << 31) && 3 * (F + 2 * n) < (1ull << 31), "%llu cuts: the mesh outgrows int32 indices",
                   (unsigned long long)n);
    PERF_CHECK_ARG(n == 0 || (d_cycles && d_third && d_vertices && d_quadrics), "NULL pointer");
    a.edges = d_cycles; a.n_edges = (int64_t)n; a.third = (int32_t*)d_third; a.pos = d_vertices; a.quad = d_quadrics;
    return dec_run<DEC_CUT>(a, (int64_t)n, stream);
}

#pragma GCC visibility pop
}
