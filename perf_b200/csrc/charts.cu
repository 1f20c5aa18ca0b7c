// charts.cu -- chart texture atlas of a triangle mesh: near-planar face clusters grown in rounds of independent merges over
// the dual graph, a planar frame per chart (the smallest of 8 rotated bounding rectangles), shelf packing of the chart
// rectangles, and exact rasterisation of the charts into texels.  The caller (ops.chart_atlas) does the sorts, scans, the
// relabelling and compaction between rounds and the density search; the library never allocates.  Every fp32 / fp64
// operation of the bodies is an explicit round-to-nearest intrinsic (never contracted), the texel geometry is fixed point and
// the only atomics are integer min / max / add, so the device build and the host build of tests/chart_harness.py
// (-DPERF_HOST_HARNESS, where each entry point runs its body over host arrays in a serial loop) agree bit for bit.
// Rules: perfb200.h (perf_chart_*); restated in numpy in tests/chart_oracle.py.
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

constexpr int64_t CHART_NO_KEY = 0x7FFFFFFFFFFFFFFFll;
constexpr int CHART_K = 8;                  // frame rotations k * 90 / 8 degrees
constexpr int CHART_GUTTER = 2;             // g: texels of margin on each side of a chart's rectangle
constexpr int CHART_FIX = 256;              // uv fixed point: 1/256 texel
constexpr double CHART_ANGLE_PAD = 1e-7;    // added to every angle: covers the acos polynomial and the rounding of the dot
constexpr double CHART_NOT_ALLOWED = 4.0;   // an "angle" above every max_angle < pi / 2

// cos, sin of k * pi / 16 (the fp64 values Python's math.cos / math.sin give)
__host__ __device__ __forceinline__ void chart_rot(int k, double& c, double& s)
{
    const double C[CHART_K] = {1.0, 0.9807852804032304, 0.9238795325112867, 0.8314696123025452, 0.7071067811865476,
                               0.5555702330196023, 0.38268343236508984, 0.19509032201612833};
    const double S[CHART_K] = {0.0, 0.19509032201612825, 0.3826834323650898, 0.5555702330196022, 0.7071067811865475,
                               0.8314696123025452, 0.9238795325112867, 0.9807852804032304};
    c = C[k]; s = S[k];
}

enum { CH_SUMS, CH_EDGES, CH_SELECT, CH_MERGE, CH_BOX, CH_FRAME, CH_RECTS, CH_NEXT, CH_LIFT, CH_START, CH_PLACE, CH_UV,
       CH_COUNT, CH_RASTER, CH_TEXELS };

struct ChartArgs {
    const float* pos; int64_t V;                        // [V,3]
    const int32_t* faces; int64_t F;                    // [F,3]
    double* S; double* alpha;                           // per chart: normal sum [.,3], cone bound
    const int32_t* edges; int64_t E;                    // dual edges [E,2]: the charts on either side
    int64_t* key; int64_t* cmin; uint8_t* sel;          // [E], per chart, [E]
    const int64_t* sel_list; double max_angle;
    const int32_t* chart; int64_t C;                    // chart of each face [F], chart count
    int64_t* box;                                       // [C, K, 4]: min x, max x, min y, max y images
    int32_t* rot; double* frame;                        // [C]: k + 8 swap; [C,4]: x0, y0, w, h
    float d; int32_t size; int32_t* rect;               // density, T; [C,4]: cw, ch, rw, rh
    const int64_t* prefix; const int32_t* height; int64_t n;   // sorted rectangles: width prefix [n + 1], heights [n]
    const int32_t* lift_in; int32_t* lift_out; int32_t* lift; int L;   // lifting table [L, n + 1]
    int32_t* start; int32_t* shelf_h;                   // [n]
    const int64_t* shelf_y; const int32_t* order; int32_t* origin;    // [n], [n] chart at each position, [C,2]
    int32_t* uvq; float* uv;                            // [F,3,2]
    int64_t* count; const int64_t* offsets; int64_t total;          // candidates per face, their inclusive scan [F + 1]
    int64_t* tkey; int32_t* inside;                     // [T^2] per texel (image order)
    const int32_t* tindex; const int32_t* tface; float* tpoint;     // [n], [n], [n,3]
};

struct D3c { double x, y, z; };

__host__ __device__ __forceinline__ D3c ch_pos(const ChartArgs& a, int32_t v)
{
    return {(double)a.pos[3 * (int64_t)v], (double)a.pos[3 * (int64_t)v + 1], (double)a.pos[3 * (int64_t)v + 2]};
}
__host__ __device__ __forceinline__ D3c ch_add(D3c a, D3c b) { return {PERF_DADD_RN(a.x, b.x), PERF_DADD_RN(a.y, b.y), PERF_DADD_RN(a.z, b.z)}; }
__host__ __device__ __forceinline__ D3c ch_sub(D3c a, D3c b) { return {PERF_DSUB_RN(a.x, b.x), PERF_DSUB_RN(a.y, b.y), PERF_DSUB_RN(a.z, b.z)}; }
__host__ __device__ __forceinline__ double ch_dot(D3c a, D3c b)
{
    return PERF_DADD_RN(PERF_DADD_RN(PERF_DMUL_RN(a.x, b.x), PERF_DMUL_RN(a.y, b.y)), PERF_DMUL_RN(a.z, b.z));
}
__host__ __device__ __forceinline__ D3c ch_load(const double* S, int64_t c) { return {S[3 * c], S[3 * c + 1], S[3 * c + 2]}; }
// S / |S|; false when S = 0
__host__ __device__ __forceinline__ bool ch_unit(D3c s, D3c& n)
{
    const double l2 = ch_dot(s, s);
    if (!(l2 > 0.0)) return false;
    const double l = PERF_DSQRT_RN(l2);
    n = {PERF_DDIV_RN(s.x, l), PERF_DDIV_RN(s.y, l), PERF_DDIV_RN(s.z, l)};
    return true;
}

// Angle between unit vectors with cosine x, padded: acos by Abramowitz & Stegun 4.4.46 (|error| <= 2e-8 on [0, 1]);
// CHART_NOT_ALLOWED for x < 0 (90 degrees or more).
__host__ __device__ __forceinline__ double ch_angle(double x)
{
    if (x < 0.0) return CHART_NOT_ALLOWED;
    if (x > 1.0) x = 1.0;
    const double A[8] = {1.5707963050, -0.2145988016, 0.0889789874, -0.0501743046, 0.0308918810, -0.0170881256, 0.0066700901,
                         -0.0012624911};
    double p = A[7];
    for (int i = 6; i >= 0; --i) p = PERF_DADD_RN(PERF_DMUL_RN(p, x), A[i]);
    return PERF_DADD_RN(PERF_DMUL_RN(PERF_DSQRT_RN(PERF_DSUB_RN(1.0, x)), p), CHART_ANGLE_PAD);
}

// Cone bound of the union of charts A and B (CHART_NOT_ALLOWED when the union's normal sum vanishes while a part's does not).
__host__ __device__ __forceinline__ double ch_merge_alpha(const ChartArgs& a, int32_t A, int32_t B)
{
    const D3c sa = ch_load(a.S, A), sb = ch_load(a.S, B);
    D3c na, nb, nab;
    const bool ha = ch_unit(sa, na), hb = ch_unit(sb, nb), hab = ch_unit(ch_add(sa, sb), nab);
    if (!hab) return (ha || hb) ? CHART_NOT_ALLOWED : 0.0;
    double r = 0.0;
    if (ha) r = PERF_DADD_RN(a.alpha[A], ch_angle(ch_dot(na, nab)));
    if (hb) { const double t = PERF_DADD_RN(a.alpha[B], ch_angle(ch_dot(nb, nab))); if (t > r) r = t; }
    return r;
}

__host__ __device__ __forceinline__ void ch_min64(int64_t* p, int64_t v)
{
#ifdef __CUDA_ARCH__
    atomicMin((long long*)p, (long long)v);
#else
    if (v < *p) *p = v;
#endif
}
__host__ __device__ __forceinline__ void ch_max64(int64_t* p, int64_t v)
{
#ifdef __CUDA_ARCH__
    atomicMax((long long*)p, (long long)v);
#else
    if (v > *p) *p = v;
#endif
}
__host__ __device__ __forceinline__ void ch_inc(int32_t* p)
{
#ifdef __CUDA_ARCH__
    atomicAdd((int*)p, 1);
#else
    ++*p;
#endif
}
// order-preserving int64 image of an fp64 value, and back
__host__ __device__ __forceinline__ int64_t ch_img(double v)
{
    int64_t b;
    memcpy(&b, &v, 8);
    return b >= 0 ? b : b ^ 0x7FFFFFFFFFFFFFFFll;
}
__host__ __device__ __forceinline__ double ch_unimg(int64_t b)
{
    b = b >= 0 ? b : b ^ 0x7FFFFFFFFFFFFFFFll;
    double v;
    memcpy(&v, &b, 8);
    return v;
}

// Face normal sum: (p1 - p0) x (p2 - p0) in fp64 (twice the area-weighted normal).
__host__ __device__ __forceinline__ void ch_sums(const ChartArgs& a, int64_t f)
{
    const D3c p0 = ch_pos(a, a.faces[3 * f]), e1 = ch_sub(ch_pos(a, a.faces[3 * f + 1]), p0), e2 = ch_sub(ch_pos(a, a.faces[3 * f + 2]), p0);
    a.S[3 * f] = PERF_DSUB_RN(PERF_DMUL_RN(e1.y, e2.z), PERF_DMUL_RN(e1.z, e2.y));
    a.S[3 * f + 1] = PERF_DSUB_RN(PERF_DMUL_RN(e1.z, e2.x), PERF_DMUL_RN(e1.x, e2.z));
    a.S[3 * f + 2] = PERF_DSUB_RN(PERF_DMUL_RN(e1.x, e2.y), PERF_DMUL_RN(e1.y, e2.x));
    a.alpha[f] = 0.0;
}

__host__ __device__ __forceinline__ void ch_edge(const ChartArgs& a, int64_t e)
{
    const int32_t A = a.edges[2 * e], B = a.edges[2 * e + 1];
    const double al = ch_merge_alpha(a, A, B);
    int64_t k = CHART_NO_KEY;
    if (al <= a.max_angle) {
        const float f = PERF_D2F_RN(al);
        uint32_t bits;
        memcpy(&bits, &f, 4);
        k = ((int64_t)bits << 32) | e;
        ch_min64(&a.cmin[A], k);
        ch_min64(&a.cmin[B], k);
    }
    a.key[e] = k;
}

__host__ __device__ __forceinline__ void ch_select(const ChartArgs& a, int64_t e)
{
    const int64_t k = a.key[e];
    a.sel[e] = k != CHART_NO_KEY && k == a.cmin[a.edges[2 * e]] && k == a.cmin[a.edges[2 * e + 1]];
}

__host__ __device__ __forceinline__ void ch_merge(const ChartArgs& a, int64_t i)
{
    const int64_t e = a.sel_list[i];
    int32_t A = a.edges[2 * e], B = a.edges[2 * e + 1];
    if (B < A) { const int32_t t = A; A = B; B = t; }
    const double al = ch_merge_alpha(a, A, B);
    for (int d = 0; d < 3; ++d) a.S[3 * (int64_t)A + d] = PERF_DADD_RN(a.S[3 * (int64_t)A + d], a.S[3 * (int64_t)B + d]);
    a.alpha[A] = al;
}

// Frame basis of chart c: n = S / |S| ((0, 0, 1) when S = 0); b1, b2 of Duff et al. 2017 (b1 x b2 = n).
__host__ __device__ __forceinline__ void ch_basis(const ChartArgs& a, int64_t c, D3c& b1, D3c& b2)
{
    D3c n;
    if (!ch_unit(ch_load(a.S, c), n)) n = {0.0, 0.0, 1.0};
    const double sg = n.z >= 0.0 ? 1.0 : -1.0;
    const double q = PERF_DDIV_RN(-1.0, PERF_DADD_RN(sg, n.z));
    const double b = PERF_DMUL_RN(PERF_DMUL_RN(n.x, n.y), q);
    b1 = {PERF_DADD_RN(1.0, PERF_DMUL_RN(PERF_DMUL_RN(PERF_DMUL_RN(sg, n.x), n.x), q)), PERF_DMUL_RN(sg, b), -PERF_DMUL_RN(sg, n.x)};
    b2 = {b, PERF_DADD_RN(sg, PERF_DMUL_RN(PERF_DMUL_RN(n.y, n.y), q)), -n.y};
}

// Rotated projection of vertex v in chart c's frame at rotation k: X = p . b1, Y = p . b2, x = c X + s Y, y = c Y - s X.
__host__ __device__ __forceinline__ void ch_project(const ChartArgs& a, int64_t c, int32_t v, int k, double& x, double& y)
{
    D3c b1, b2;
    ch_basis(a, c, b1, b2);
    const D3c p = ch_pos(a, v);
    const double X = ch_dot(p, b1), Y = ch_dot(p, b2);
    double cs, sn;
    chart_rot(k, cs, sn);
    x = PERF_DADD_RN(PERF_DMUL_RN(cs, X), PERF_DMUL_RN(sn, Y));
    y = PERF_DSUB_RN(PERF_DMUL_RN(cs, Y), PERF_DMUL_RN(sn, X));
}

__host__ __device__ __forceinline__ void ch_box(const ChartArgs& a, int64_t i)
{
    const int64_t c = a.chart[i / 3];
    const int32_t v = a.faces[i];
    for (int k = 0; k < CHART_K; ++k) {
        double x, y;
        ch_project(a, c, v, k, x, y);
        int64_t* b = a.box + 4 * (CHART_K * c + k);
        ch_min64(b, ch_img(x)); ch_max64(b + 1, ch_img(x)); ch_min64(b + 2, ch_img(y)); ch_max64(b + 3, ch_img(y));
    }
}

// Rotation of the smallest rectangle area (w h, the first k on a tie), turned to landscape by (x, y) -> (y, -x) when h > w.
__host__ __device__ __forceinline__ void ch_frame(const ChartArgs& a, int64_t c)
{
    int best = 0;
    double bx0 = 0, bx1 = 0, by0 = 0, by1 = 0, barea = 0;
    for (int k = 0; k < CHART_K; ++k) {
        const int64_t* b = a.box + 4 * (CHART_K * c + k);
        const double x0 = ch_unimg(b[0]), x1 = ch_unimg(b[1]), y0 = ch_unimg(b[2]), y1 = ch_unimg(b[3]);
        const double ar = PERF_DMUL_RN(PERF_DSUB_RN(x1, x0), PERF_DSUB_RN(y1, y0));
        if (k == 0 || ar < barea) { best = k; barea = ar; bx0 = x0; bx1 = x1; by0 = y0; by1 = y1; }
    }
    const double w = PERF_DSUB_RN(bx1, bx0), h = PERF_DSUB_RN(by1, by0);
    double* fr = a.frame + 4 * c;
    if (h > w) { a.rot[c] = best + CHART_K; fr[0] = by0; fr[1] = -bx1; fr[2] = h; fr[3] = w; }
    else { a.rot[c] = best; fr[0] = bx0; fr[1] = by0; fr[2] = w; fr[3] = h; }
}

// Chart side in texels at density d: max(1, ceil(ext d)), capped at 2^24; the rectangle adds 2g.
__host__ __device__ __forceinline__ int32_t ch_cells(double ext, float d)
{
    const double e = PERF_DMUL_RN(ext, (double)d);
    if (!(e > 1.0)) return 1;
    if (e > 16777216.0) return 16777216;
    return (int32_t)ceil(e);
}
__host__ __device__ __forceinline__ void ch_rect(const ChartArgs& a, int64_t c)
{
    const int32_t cw = ch_cells(a.frame[4 * c + 2], a.d), chh = ch_cells(a.frame[4 * c + 3], a.d);
    int32_t* r = a.rect + 4 * c;
    r[0] = cw; r[1] = chh; r[2] = cw + 2 * CHART_GUTTER; r[3] = chh + 2 * CHART_GUTTER;
}

// next[i]: the largest j <= n with prefix[j] - prefix[i] <= T (the first rectangle of the next shelf); next[n] = n.
__host__ __device__ __forceinline__ void ch_next(const ChartArgs& a, int64_t i)
{
    const int64_t lim = a.prefix[i] + a.size;
    int64_t lo = i, hi = a.n + 1;                       // prefix[lo] <= lim < prefix[hi] (prefix[n + 1] = +inf)
    while (hi - lo > 1) {
        const int64_t mid = (lo + hi) >> 1;
        if (a.prefix[mid] <= lim) lo = mid; else hi = mid;
    }
    a.lift_out[i] = (int32_t)lo;
}

__host__ __device__ __forceinline__ void ch_lift(const ChartArgs& a, int64_t i) { a.lift_out[i] = a.lift_in[a.lift_in[i]]; }

// Shelf k starts at next^k(0) (n when there are fewer shelves); its height is that of its first (tallest) rectangle.
__host__ __device__ __forceinline__ void ch_start(const ChartArgs& a, int64_t k)
{
    int64_t i = 0;
    for (int l = 0; l < a.L && i < a.n; ++l)
        if ((k >> l) & 1) i = a.lift[(int64_t)l * (a.n + 1) + i];
    a.start[k] = (int32_t)i;
    a.shelf_h[k] = i < a.n ? a.height[i] : 0;
}

// Rectangle at sorted position i: its shelf k (the last start <= i), x = prefix[i] - prefix[start_k], y = shelf_y[k].
__host__ __device__ __forceinline__ void ch_place(const ChartArgs& a, int64_t i)
{
    int64_t lo = 0, hi = a.n;                           // start[lo] <= i < start[hi]
    while (hi - lo > 1) {
        const int64_t mid = (lo + hi) >> 1;
        if (a.start[mid] <= i) lo = mid; else hi = mid;
    }
    const int32_t c = a.order[i];
    a.origin[2 * (int64_t)c] = (int32_t)(a.prefix[i] - a.prefix[a.start[lo]]);
    a.origin[2 * (int64_t)c + 1] = (int32_t)a.shelf_y[lo];
}

// Corner uv in fixed point: per axis q = clamp(floor((local d) 256 + 0.5), 0, 256 cells), U = 256 (origin + g) + q.
__host__ __device__ __forceinline__ int32_t ch_fix(double local, float d, int32_t cells, int32_t o)
{
    const double t = PERF_DADD_RN(PERF_DMUL_RN(PERF_DMUL_RN(local, (double)d), (double)CHART_FIX), 0.5);
    double q = floor(t);
    const double qmax = (double)cells * CHART_FIX;
    q = q < 0.0 ? 0.0 : (q > qmax ? qmax : q);
    return CHART_FIX * (o + CHART_GUTTER) + (int32_t)q;
}
__host__ __device__ __forceinline__ void ch_uv(const ChartArgs& a, int64_t i)
{
    const int64_t c = a.chart[i / 3];
    const int32_t r = a.rot[c];
    double x, y;
    ch_project(a, c, a.faces[i], r % CHART_K, x, y);
    if (r >= CHART_K) { const double t = x; x = y; y = -t; }
    const double* fr = a.frame + 4 * c;
    const int32_t* rc = a.rect + 4 * c;
    const int32_t U = ch_fix(PERF_DSUB_RN(x, fr[0]), a.d, rc[0], a.origin[2 * c]);
    const int32_t W = ch_fix(PERF_DSUB_RN(y, fr[1]), a.d, rc[1], a.origin[2 * c + 1]);
    a.uvq[2 * i] = U; a.uvq[2 * i + 1] = W;
    const float den = (float)CHART_FIX * (float)a.size;
    a.uv[2 * i] = PERF_FDIV_RN((float)U, den);
    a.uv[2 * i + 1] = PERF_FDIV_RN((float)W, den);
}

__host__ __device__ __forceinline__ int64_t ch_floordiv(int64_t a, int64_t b) { return a >= 0 ? a / b : -((-a + b - 1) / b); }

// Candidate texels of face f: texel x (centre 256 x + 128) with 256 x + 128 in [min U - 256 g, max U + 256 g], clamped to the texture.
__host__ __device__ __forceinline__ void ch_range(const ChartArgs& a, int64_t f, int32_t& x0, int32_t& x1, int32_t& y0, int32_t& y1)
{
    const int32_t* q = a.uvq + 6 * f;
    int32_t u0 = q[0], u1 = q[0], v0 = q[1], v1 = q[1];
    for (int k = 1; k < 3; ++k) {
        u0 = q[2 * k] < u0 ? q[2 * k] : u0; u1 = q[2 * k] > u1 ? q[2 * k] : u1;
        v0 = q[2 * k + 1] < v0 ? q[2 * k + 1] : v0; v1 = q[2 * k + 1] > v1 ? q[2 * k + 1] : v1;
    }
    const int32_t m = CHART_FIX * CHART_GUTTER, h = CHART_FIX / 2;
    x0 = (int32_t)-ch_floordiv(-(int64_t)(u0 - m - h), CHART_FIX); x1 = (int32_t)ch_floordiv(u1 + m - h, CHART_FIX);
    y0 = (int32_t)-ch_floordiv(-(int64_t)(v0 - m - h), CHART_FIX); y1 = (int32_t)ch_floordiv(v1 + m - h, CHART_FIX);
    x0 = x0 < 0 ? 0 : x0; y0 = y0 < 0 ? 0 : y0;
    x1 = x1 > a.size - 1 ? a.size - 1 : x1; y1 = y1 > a.size - 1 ? a.size - 1 : y1;
}

__host__ __device__ __forceinline__ void ch_count(const ChartArgs& a, int64_t f)
{
    int32_t x0, x1, y0, y1;
    ch_range(a, f, x0, x1, y0, y1);
    a.count[f] = (x1 < x0 || y1 < y0) ? 0 : (int64_t)(x1 - x0 + 1) * (y1 - y0 + 1);
}

// Texel centre P (fixed point) against face f: inside (edge functions, top-left rule, positive area) or the nearest point of
// the three edges (fp64, strictly nearer wins, edges 0-1, 1-2, 2-0).  Returns inside; dist2 and the edge / parameter.
__host__ __device__ __forceinline__ bool ch_locate(const ChartArgs& a, int64_t f, int64_t px, int64_t py, int64_t (&w)[3], int64_t& area,
                                                   double& dist2, int& edge, double& t)
{
    const int32_t* q = a.uvq + 6 * f;
    int64_t X[3], Y[3];
    for (int k = 0; k < 3; ++k) { X[k] = q[2 * k]; Y[k] = q[2 * k + 1]; }
    area = (X[1] - X[0]) * (Y[2] - Y[0]) - (Y[1] - Y[0]) * (X[2] - X[0]);
    bool in = area > 0;
    for (int k = 0; k < 3; ++k) {                       // w[k]: edge k+1 -> k+2 (opposite corner k)
        const int i = (k + 1) % 3, j = (k + 2) % 3;
        const int64_t dx = X[j] - X[i], dy = Y[j] - Y[i];
        w[k] = dx * (py - Y[i]) - dy * (px - X[i]);
        const bool tl = dy < 0 || (dy == 0 && dx < 0);
        in = in && (w[k] > 0 || (w[k] == 0 && tl));
    }
    if (in) { dist2 = 0.0; edge = -1; t = 0.0; return true; }
    dist2 = -1.0;
    for (int k = 0; k < 3; ++k) {
        const int j = (k + 1) % 3;
        const double ax = (double)X[k], ay = (double)Y[k], dx = (double)(X[j] - X[k]), dy = (double)(Y[j] - Y[k]);
        const double rx = PERF_DSUB_RN((double)px, ax), ry = PERF_DSUB_RN((double)py, ay);
        const double dd = PERF_DADD_RN(PERF_DMUL_RN(dx, dx), PERF_DMUL_RN(dy, dy));
        double s = 0.0;
        if (dd > 0.0) {
            s = PERF_DDIV_RN(PERF_DADD_RN(PERF_DMUL_RN(rx, dx), PERF_DMUL_RN(ry, dy)), dd);
            s = s < 0.0 ? 0.0 : (s > 1.0 ? 1.0 : s);
        }
        const double ex = PERF_DSUB_RN(rx, PERF_DMUL_RN(s, dx)), ey = PERF_DSUB_RN(ry, PERF_DMUL_RN(s, dy));
        const double d2 = PERF_DADD_RN(PERF_DMUL_RN(ex, ex), PERF_DMUL_RN(ey, ey));
        if (dist2 < 0.0 || d2 < dist2) { dist2 = d2; edge = k; t = s; }
    }
    return false;
}

__host__ __device__ __forceinline__ void ch_raster(const ChartArgs& a, int64_t j)
{
    int64_t lo = 0, hi = a.F;                           // offsets[lo] <= j < offsets[hi]  (offsets[0] = 0)
    while (hi - lo > 1) {
        const int64_t mid = (lo + hi) >> 1;
        if (a.offsets[mid] <= j) lo = mid; else hi = mid;
    }
    const int64_t f = lo;
    int32_t x0, x1, y0, y1;
    ch_range(a, f, x0, x1, y0, y1);
    const int64_t local = j - a.offsets[f], nx = x1 - x0 + 1;
    const int64_t x = x0 + local % nx, y = y0 + local / nx;
    int64_t w[3], area;
    double d2, t;
    int edge;
    const bool in = ch_locate(a, f, CHART_FIX * x + CHART_FIX / 2, CHART_FIX * y + CHART_FIX / 2, w, area, d2, edge, t);
    const double g = (double)(CHART_FIX * CHART_GUTTER);
    if (!in && !(d2 <= PERF_DMUL_RN(g, g))) return;
    const int64_t m = (a.size - 1 - y) * (int64_t)a.size + x;
    int64_t key = f;
    if (!in) {
        const float fd = PERF_D2F_RN(d2);
        uint32_t bits;
        memcpy(&bits, &fd, 4);
        key |= (int64_t)(bits + 1u) << 32;
    } else {
        ch_inc(&a.inside[m]);
    }
    ch_min64(&a.tkey[m], key);
}

// World point of used texel i: inside -> barycentrics w / area (fp64, then fp32), p = (p0 + b1 (p1 - p0)) + b2 (p2 - p0);
// else the nearest edge point, p = pk + t (pk+1 - pk) with t rounded to fp32.
__host__ __device__ __forceinline__ void ch_texel(const ChartArgs& a, int64_t i)
{
    const int64_t m = a.tindex[i], f = a.tface[i];
    const int64_t x = m % a.size, y = a.size - 1 - m / a.size;
    int64_t w[3], area;
    double d2, t;
    int edge;
    const bool in = ch_locate(a, f, CHART_FIX * x + CHART_FIX / 2, CHART_FIX * y + CHART_FIX / 2, w, area, d2, edge, t);
    float p[3][3];
    for (int k = 0; k < 3; ++k)
        for (int d = 0; d < 3; ++d) p[k][d] = a.pos[3 * (int64_t)a.faces[3 * f + k] + d];
    float* out = a.tpoint + 3 * i;
    if (in) {
        const float b1 = PERF_D2F_RN(PERF_DDIV_RN((double)w[1], (double)area)), b2 = PERF_D2F_RN(PERF_DDIV_RN((double)w[2], (double)area));
        for (int d = 0; d < 3; ++d)
            out[d] = PERF_FADD_RN(PERF_FADD_RN(p[0][d], PERF_FMUL_RN(b1, PERF_FSUB_RN(p[1][d], p[0][d]))),
                                  PERF_FMUL_RN(b2, PERF_FSUB_RN(p[2][d], p[0][d])));
    } else {
        const float tf = PERF_D2F_RN(t);
        const int k = edge, j = (edge + 1) % 3;
        for (int d = 0; d < 3; ++d) out[d] = PERF_FADD_RN(p[k][d], PERF_FMUL_RN(tf, PERF_FSUB_RN(p[j][d], p[k][d])));
    }
}

template <int S>
__host__ __device__ __forceinline__ void chart_body(const ChartArgs& a, int64_t i)
{
    if (S == CH_SUMS) ch_sums(a, i);
    else if (S == CH_EDGES) ch_edge(a, i);
    else if (S == CH_SELECT) ch_select(a, i);
    else if (S == CH_MERGE) ch_merge(a, i);
    else if (S == CH_BOX) ch_box(a, i);
    else if (S == CH_FRAME) ch_frame(a, i);
    else if (S == CH_RECTS) ch_rect(a, i);
    else if (S == CH_NEXT) ch_next(a, i);
    else if (S == CH_LIFT) ch_lift(a, i);
    else if (S == CH_START) ch_start(a, i);
    else if (S == CH_PLACE) ch_place(a, i);
    else if (S == CH_UV) ch_uv(a, i);
    else if (S == CH_COUNT) ch_count(a, i);
    else if (S == CH_RASTER) ch_raster(a, i);
    else ch_texel(a, i);
}

template <int S>
__global__ void __launch_bounds__(128) chart_kernel(const ChartArgs a, int64_t n)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) chart_body<S>(a, i);
}

// The product library launches the kernel; the test harness build runs the same body over host arrays.
template <int S>
static int chart_run(const ChartArgs& a, int64_t n, void* stream)
{
    if (n <= 0) return PERF_OK;
#ifdef PERF_HOST_HARNESS
    (void)stream;
    for (int64_t i = 0; i < n; ++i) chart_body<S>(a, i);
#else
    chart_kernel<S><<<(unsigned)((n + 127) / 128), 128, 0, (cudaStream_t)stream>>>(a, n);
    PERF_LAUNCH_CHECK();
#endif
    return PERF_OK;
}

}  // namespace perf

using namespace perf;

static int chart_fill(ChartArgs& a, const float* vertices, uint64_t V, const int32_t* faces, uint64_t F)
{
    PERF_CHECK_ARG(V < (1ull << 31) && F < (1ull << 29), "mesh of %llu vertices / %llu faces: needs V < 2^31 and F < 2^29",
                   (unsigned long long)V, (unsigned long long)F);
    PERF_CHECK_ARG(F == 0 || faces, "NULL faces");
    memset(&a, 0, sizeof(a));
    a.pos = vertices; a.V = (int64_t)V; a.faces = faces; a.F = (int64_t)F;
    return PERF_OK;
}

#define CHART_SIZE_OK(T) ((T) >= 256 && (T) <= 16384 && ((T) & ((T) - 1)) == 0)

extern "C" {
#pragma GCC visibility push(default)

int perf_chart_sums(const float* d_vertices, uint64_t V, const int32_t* d_faces, uint64_t F, double* d_sums, double* d_alpha, void* stream)
{
    ChartArgs a;
    int rc = chart_fill(a, d_vertices, V, d_faces, F); if (rc) return rc;
    PERF_CHECK_ARG(F == 0 || (d_vertices && d_sums && d_alpha), "NULL pointer");
    a.S = d_sums; a.alpha = d_alpha;
    return chart_run<CH_SUMS>(a, (int64_t)F, stream);
}

int perf_chart_edges(const int32_t* d_edges, uint64_t E, const double* d_sums, const double* d_alpha, double max_angle, int64_t* d_key,
                     int64_t* d_cmin, void* stream)
{
    ChartArgs a;
    memset(&a, 0, sizeof(a));
    PERF_CHECK_ARG(E < (1ull << 31), "%llu dual edges", (unsigned long long)E);
    PERF_CHECK_ARG(max_angle > 0.0 && max_angle < 1.5707963267948966, "max_angle %g: needs (0, pi/2) radians", max_angle);
    PERF_CHECK_ARG(E == 0 || (d_edges && d_sums && d_alpha && d_key && d_cmin), "NULL pointer");
    a.edges = d_edges; a.E = (int64_t)E; a.S = (double*)d_sums; a.alpha = (double*)d_alpha; a.max_angle = max_angle; a.key = d_key; a.cmin = d_cmin;
    return chart_run<CH_EDGES>(a, (int64_t)E, stream);
}

int perf_chart_select(const int32_t* d_edges, uint64_t E, const int64_t* d_key, const int64_t* d_cmin, uint8_t* d_selected, void* stream)
{
    ChartArgs a;
    memset(&a, 0, sizeof(a));
    PERF_CHECK_ARG(E < (1ull << 31), "%llu dual edges", (unsigned long long)E);
    PERF_CHECK_ARG(E == 0 || (d_edges && d_key && d_cmin && d_selected), "NULL pointer");
    a.edges = d_edges; a.E = (int64_t)E; a.key = (int64_t*)d_key; a.cmin = (int64_t*)d_cmin; a.sel = d_selected;
    return chart_run<CH_SELECT>(a, (int64_t)E, stream);
}

int perf_chart_merge(const int32_t* d_edges, const int64_t* d_selected_ids, uint64_t n, double* d_sums, double* d_alpha, void* stream)
{
    ChartArgs a;
    memset(&a, 0, sizeof(a));
    PERF_CHECK_ARG(n == 0 || (d_edges && d_selected_ids && d_sums && d_alpha), "NULL pointer");
    a.edges = d_edges; a.sel_list = d_selected_ids; a.S = d_sums; a.alpha = d_alpha;
    return chart_run<CH_MERGE>(a, (int64_t)n, stream);
}

int perf_chart_frames(const float* d_vertices, uint64_t V, const int32_t* d_faces, uint64_t F, const int32_t* d_chart, uint64_t C,
                      const double* d_sums, int64_t* d_box, int32_t* d_rot, double* d_frame, void* stream)
{
    ChartArgs a;
    int rc = chart_fill(a, d_vertices, V, d_faces, F); if (rc) return rc;
    PERF_CHECK_ARG(C <= F, "%llu charts of %llu faces", (unsigned long long)C, (unsigned long long)F);
    PERF_CHECK_ARG(F == 0 || (d_vertices && d_chart && d_sums && d_box && d_rot && d_frame), "NULL pointer");
    a.chart = d_chart; a.C = (int64_t)C; a.S = (double*)d_sums; a.box = d_box; a.rot = d_rot; a.frame = d_frame;
    rc = chart_run<CH_BOX>(a, 3 * (int64_t)F, stream); if (rc) return rc;
    return chart_run<CH_FRAME>(a, (int64_t)C, stream);
}

int perf_chart_rects(const double* d_frame, uint64_t C, float density, int32_t* d_rect, void* stream)
{
    ChartArgs a;
    memset(&a, 0, sizeof(a));
    PERF_CHECK_ARG(density >= 0.0f && density < INFINITY, "density %g", (double)density);
    PERF_CHECK_ARG(C == 0 || (d_frame && d_rect), "NULL pointer");
    a.frame = (double*)d_frame; a.C = (int64_t)C; a.d = density; a.rect = d_rect;
    return chart_run<CH_RECTS>(a, (int64_t)C, stream);
}

int perf_chart_shelves(const int64_t* d_prefix, const int32_t* d_height, uint64_t n, int size, int32_t* d_lift, int levels,
                       int32_t* d_start, int32_t* d_shelf_h, void* stream)
{
    ChartArgs a;
    memset(&a, 0, sizeof(a));
    PERF_CHECK_ARG(CHART_SIZE_OK(size), "texture size %d: needs a power of two in [256, 16384]", size);
    PERF_CHECK_ARG(n < (1ull << 30) && levels >= 1 && levels <= 31 && (n >> (levels - 1)) <= 1, "%llu rectangles, %d levels",
                   (unsigned long long)n, levels);
    PERF_CHECK_ARG(n == 0 || (d_prefix && d_height && d_lift && d_start && d_shelf_h), "NULL pointer");
    a.prefix = d_prefix; a.height = d_height; a.n = (int64_t)n; a.size = size; a.lift = d_lift; a.L = levels;
    a.start = d_start; a.shelf_h = d_shelf_h;
    if (n == 0) return PERF_OK;
    a.lift_out = d_lift;
    int rc = chart_run<CH_NEXT>(a, (int64_t)n + 1, stream); if (rc) return rc;
    for (int l = 1; l < levels; ++l) {
        a.lift_in = d_lift + (int64_t)(l - 1) * (int64_t)(n + 1);
        a.lift_out = d_lift + (int64_t)l * (int64_t)(n + 1);
        rc = chart_run<CH_LIFT>(a, (int64_t)n + 1, stream); if (rc) return rc;
    }
    return chart_run<CH_START>(a, (int64_t)n, stream);
}

int perf_chart_place(const int64_t* d_prefix, const int32_t* d_start, const int64_t* d_shelf_y, const int32_t* d_order, uint64_t n,
                     int32_t* d_origin, void* stream)
{
    ChartArgs a;
    memset(&a, 0, sizeof(a));
    PERF_CHECK_ARG(n < (1ull << 30), "%llu rectangles", (unsigned long long)n);
    PERF_CHECK_ARG(n == 0 || (d_prefix && d_start && d_shelf_y && d_order && d_origin), "NULL pointer");
    a.prefix = d_prefix; a.start = (int32_t*)d_start; a.shelf_y = d_shelf_y; a.order = d_order; a.n = (int64_t)n; a.origin = d_origin;
    return chart_run<CH_PLACE>(a, (int64_t)n, stream);
}

int perf_chart_uv(const float* d_vertices, uint64_t V, const int32_t* d_faces, uint64_t F, const int32_t* d_chart, uint64_t C,
                  const double* d_sums, const int32_t* d_rot, const double* d_frame, const int32_t* d_rect, const int32_t* d_origin,
                  float density, int size, int32_t* d_uvq, float* d_uv, void* stream)
{
    ChartArgs a;
    int rc = chart_fill(a, d_vertices, V, d_faces, F); if (rc) return rc;
    PERF_CHECK_ARG(CHART_SIZE_OK(size), "texture size %d: needs a power of two in [256, 16384]", size);
    PERF_CHECK_ARG(C <= F && density >= 0.0f && density < INFINITY, "%llu charts, density %g", (unsigned long long)C, (double)density);
    PERF_CHECK_ARG(F == 0 || (d_vertices && d_chart && d_sums && d_rot && d_frame && d_rect && d_origin && d_uvq && d_uv), "NULL pointer");
    a.chart = d_chart; a.C = (int64_t)C; a.S = (double*)d_sums; a.rot = (int32_t*)d_rot; a.frame = (double*)d_frame;
    a.rect = (int32_t*)d_rect; a.origin = (int32_t*)d_origin; a.d = density; a.size = size; a.uvq = d_uvq; a.uv = d_uv;
    return chart_run<CH_UV>(a, 3 * (int64_t)F, stream);
}

int perf_chart_count(const int32_t* d_uvq, uint64_t F, int size, int64_t* d_count, void* stream)
{
    ChartArgs a;
    memset(&a, 0, sizeof(a));
    PERF_CHECK_ARG(CHART_SIZE_OK(size) && F < (1ull << 29), "texture size %d, %llu faces", size, (unsigned long long)F);
    PERF_CHECK_ARG(F == 0 || (d_uvq && d_count), "NULL pointer");
    a.uvq = (int32_t*)d_uvq; a.F = (int64_t)F; a.size = size; a.count = d_count;
    return chart_run<CH_COUNT>(a, (int64_t)F, stream);
}

int perf_chart_raster(const int32_t* d_uvq, uint64_t F, int size, const int64_t* d_offsets, uint64_t total, int64_t* d_key,
                      int32_t* d_inside, void* stream)
{
    ChartArgs a;
    memset(&a, 0, sizeof(a));
    PERF_CHECK_ARG(CHART_SIZE_OK(size) && F < (1ull << 29), "texture size %d, %llu faces", size, (unsigned long long)F);
    PERF_CHECK_ARG(total == 0 || (d_uvq && d_offsets && d_key && d_inside), "NULL pointer");
    a.uvq = (int32_t*)d_uvq; a.F = (int64_t)F; a.size = size; a.offsets = d_offsets; a.total = (int64_t)total; a.tkey = d_key; a.inside = d_inside;
    return chart_run<CH_RASTER>(a, (int64_t)total, stream);
}

int perf_chart_texels(const float* d_vertices, uint64_t V, const int32_t* d_faces, uint64_t F, const int32_t* d_uvq, int size,
                      const int32_t* d_index, const int32_t* d_face, uint64_t n, float* d_point, void* stream)
{
    ChartArgs a;
    int rc = chart_fill(a, d_vertices, V, d_faces, F); if (rc) return rc;
    PERF_CHECK_ARG(CHART_SIZE_OK(size), "texture size %d: needs a power of two in [256, 16384]", size);
    PERF_CHECK_ARG(n == 0 || (d_vertices && d_uvq && d_index && d_face && d_point), "NULL pointer");
    a.uvq = (int32_t*)d_uvq; a.size = size; a.tindex = d_index; a.tface = d_face; a.tpoint = d_point;
    return chart_run<CH_TEXELS>(a, (int64_t)n, stream);
}

#pragma GCC visibility pop
}
