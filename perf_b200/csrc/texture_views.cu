// texture_views.cu -- colour of texel points from registered panoramas: per texel point, a depth-tested bilinear projection
// into every view in registration order, blended with weights cos(theta) / dist^2.  Every fp32 operation is an explicit
// round-to-nearest intrinsic and atan2 is a polynomial of such operations, so the device build and the host build of
// tests/texture_views_harness.py (-DPERF_HOST_HARNESS, the body run over host arrays in a serial loop) agree bit for bit.
// Rules: perfb200.h (perf_texture_views); restated in numpy in tests/texture_views_oracle.py.
#include "common.cuh"

#ifdef __CUDA_ARCH__
#define PERF_FSQRT_RN(a) __fsqrt_rn(a)
#else
#define PERF_FSQRT_RN(a) sqrtf(a)
#endif

namespace perf {

constexpr int VIEWS_MAX = 64;
constexpr float VIEWS_MIN_COS = 0.15f;          // sup_info.py's grazing limit (normal_cos > 0.15)

struct ViewsArgs {
    const float* points; const int32_t* face; int64_t N;     // [N,3], [N]
    const float* fnormal; int64_t F;                         // [F,3]
    const float4* views; int n_views, H, W;                  // [n_views,H,W]: r, g, b, distance
    float rot[VIEWS_MAX][9]; float cen[VIEWS_MAX][3];        // camera-to-world rotation (row-major) and centre per view
    float tol;
    float* rgb; float* weight; int32_t* view;                // [N,3], [N], [N]
};

// atan2(y, x) in fp32 from rounded operations: t = min(|x|, |y|) / max(|x|, |y|) in [0, 1]; above tan(pi/8) t is reduced
// to (t - 1) / (t + 1) (pi/4 added back); atan(t) = t + (t s) q(s), s = t t, q a degree-3 polynomial in Horner form; then
// the octant and quadrant reflections.  atan2(0, 0) = 0.  Max |error| against fp64 arctan2: perfb200.h.
__host__ __device__ __forceinline__ float views_atan2(float y, float x)
{
    const float ax = fabsf(x), ay = fabsf(y);
    const float mx = fmaxf(ax, ay), mn = fminf(ax, ay);
    if (!(mx > 0.0f)) return 0.0f;
    float t = PERF_FDIV_RN(mn, mx);
    const bool big = t > 0.41421356f;
    if (big) t = PERF_FDIV_RN(PERF_FSUB_RN(t, 1.0f), PERF_FADD_RN(t, 1.0f));
    const float s = PERF_FMUL_RN(t, t);
    float q = 0.08037880063056946f;
    q = PERF_FADD_RN(-0.13872261345386505f, PERF_FMUL_RN(s, q));
    q = PERF_FADD_RN(0.19977140426635742f, PERF_FMUL_RN(s, q));
    q = PERF_FADD_RN(-0.33332931995391846f, PERF_FMUL_RN(s, q));
    float r = PERF_FADD_RN(t, PERF_FMUL_RN(PERF_FMUL_RN(t, s), q));
    if (big) r = PERF_FADD_RN(0.785398185253143310546875f, r);          // fp32(pi / 4)
    if (ay > ax) r = PERF_FSUB_RN(1.57079637050628662109375f, r);        // fp32(pi / 2)
    if (x < 0.0f) r = PERF_FSUB_RN(3.14159274101257324f, r);             // fp32(pi)
    return y < 0.0f ? -r : r;
}

__host__ __device__ __forceinline__ float views_dot(const float* a, const float* b)
{
    return PERF_FADD_RN(PERF_FADD_RN(PERF_FMUL_RN(a[0], b[0]), PERF_FMUL_RN(a[1], b[1])), PERF_FMUL_RN(a[2], b[2]));
}

// Texel point i against every view in order (perfb200.h states the rule step by step).
__host__ __device__ __forceinline__ void views_texel(const ViewsArgs& a, int64_t i)
{
    const int32_t f = a.face[i];
    if (f < 0) {
        for (int d = 0; d < 3; ++d) a.rgb[3 * i + d] = 0.0f;
        a.weight[i] = 0.0f; a.view[i] = -2;
        return;
    }
    const float p[3] = {a.points[3 * i], a.points[3 * i + 1], a.points[3 * i + 2]};
    const float n[3] = {a.fnormal[3 * (int64_t)f], a.fnormal[3 * (int64_t)f + 1], a.fnormal[3 * (int64_t)f + 2]};
    const float Wf = (float)a.W, Hf = (float)a.H;
    float acc[3] = {0.0f, 0.0f, 0.0f}, wsum = 0.0f, best = 0.0f;
    int32_t best_v = -1;
    for (int v = 0; v < a.n_views; ++v) {
        const float* R = a.rot[v];
        const float q[3] = {PERF_FSUB_RN(p[0], a.cen[v][0]), PERF_FSUB_RN(p[1], a.cen[v][1]), PERF_FSUB_RN(p[2], a.cen[v][2])};
        const float dist2 = views_dot(q, q);
        if (!(dist2 > 0.0f)) continue;
        const float dist = PERF_FSQRT_RN(dist2);
        const float cosv = PERF_FDIV_RN(-views_dot(n, q), dist);            // n . (c - p) / dist
        if (!(cosv >= VIEWS_MIN_COS)) continue;
        float c[3];                                                         // R^T q / dist
        for (int d = 0; d < 3; ++d)
            c[d] = PERF_FDIV_RN(PERF_FADD_RN(PERF_FADD_RN(PERF_FMUL_RN(R[d], q[0]), PERF_FMUL_RN(R[3 + d], q[1])),
                                             PERF_FMUL_RN(R[6 + d], q[2])), dist);
        const float alpha = views_atan2(c[1], c[0]);
        const float beta = views_atan2(c[2], PERF_FSQRT_RN(PERF_FADD_RN(PERF_FMUL_RN(c[0], c[0]), PERF_FMUL_RN(c[1], c[1]))));
        const float x = PERF_FSUB_RN(PERF_FMUL_RN(PERF_FSUB_RN(0.5f, PERF_FMUL_RN(alpha, 0.159154937f)), Wf), 0.5f);   // 1 / 2pi
        const float y = PERF_FSUB_RN(PERF_FMUL_RN(PERF_FSUB_RN(0.5f, PERF_FMUL_RN(beta, 0.318309873f)), Hf), 0.5f);    // 1 / pi
        const float x0 = floorf(x), y0 = floorf(y);
        const float fx = PERF_FSUB_RN(x, x0), fy = PERF_FSUB_RN(y, y0);
        const float gx = PERF_FSUB_RN(1.0f, fx), gy = PERF_FSUB_RN(1.0f, fy);
        int32_t c0 = (int32_t)x0 % a.W;
        if (c0 < 0) c0 += a.W;
        const int32_t cols[2] = {c0, c0 + 1 == a.W ? 0 : c0 + 1};
        const int32_t r0 = (int32_t)y0;
        const int32_t rows[2] = {r0 < 0 ? 0 : (r0 > a.H - 1 ? a.H - 1 : r0), r0 + 1 < 0 ? 0 : (r0 + 1 > a.H - 1 ? a.H - 1 : r0 + 1)};
        const float4* img = a.views + (int64_t)v * a.H * a.W;
        float s[3] = {0.0f, 0.0f, 0.0f}, sw = 0.0f;
        for (int k = 0; k < 4; ++k) {                                       // taps (x0, y0), (x0 + 1, y0), (x0, y0 + 1), (x0 + 1, y0 + 1)
            const float w = PERF_FMUL_RN((k & 1) ? fx : gx, (k & 2) ? fy : gy);
            const float4 t = img[(int64_t)rows[k >> 1] * a.W + cols[k & 1]];
            if (!(w > 0.0f && t.w > 0.0f && fabsf(PERF_FSUB_RN(dist, t.w)) <= a.tol)) continue;
            s[0] = PERF_FADD_RN(s[0], PERF_FMUL_RN(w, t.x));
            s[1] = PERF_FADD_RN(s[1], PERF_FMUL_RN(w, t.y));
            s[2] = PERF_FADD_RN(s[2], PERF_FMUL_RN(w, t.z));
            sw = PERF_FADD_RN(sw, w);
        }
        if (!(sw > 0.0f)) continue;
        const float wv = PERF_FDIV_RN(cosv, dist2);
        for (int d = 0; d < 3; ++d) acc[d] = PERF_FADD_RN(acc[d], PERF_FMUL_RN(wv, PERF_FDIV_RN(s[d], sw)));
        wsum = PERF_FADD_RN(wsum, wv);
        if (wv > best) { best = wv; best_v = v; }
    }
    for (int d = 0; d < 3; ++d) a.rgb[3 * i + d] = wsum > 0.0f ? PERF_FDIV_RN(acc[d], wsum) : 0.0f;
    a.weight[i] = wsum; a.view[i] = best_v;
}

__global__ void __launch_bounds__(128) views_kernel(const ViewsArgs a)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < a.N) views_texel(a, i);
}

}  // namespace perf

using namespace perf;

extern "C" {
#pragma GCC visibility push(default)

int perf_texture_views(const float* d_points, const int32_t* d_face, uint64_t N, const float* d_face_normal, uint64_t F,
                       const float* d_views, int n_views, int H, int W, const float* h_poses, float depth_tol, float* d_rgb,
                       float* d_weight, int32_t* d_view, void* stream)
{
    PERF_CHECK_ARG(n_views >= 0 && n_views <= VIEWS_MAX, "%d views: at most %d", n_views, VIEWS_MAX);
    PERF_CHECK_ARG(n_views == 0 || (H >= 1 && W >= 1 && (int64_t)H * W < (1ll << 31)), "view size %d x %d", H, W);
    PERF_CHECK_ARG(N < (1ull << 40) && F < (1ull << 31), "%llu texel points / %llu faces", (unsigned long long)N, (unsigned long long)F);
    PERF_CHECK_ARG(N == 0 || (d_points && d_face && d_rgb && d_weight && d_view), "NULL pointer");
    PERF_CHECK_ARG(n_views == 0 || (d_views && h_poses && ((uintptr_t)d_views & 15) == 0), "views: NULL or not 16-byte aligned");
    PERF_CHECK_ARG(F == 0 || d_face_normal, "NULL face normals");
    PERF_CHECK_ARG(depth_tol >= 0.0f, "depth_tol %g: needs >= 0", (double)depth_tol);
    ViewsArgs a;
    memset(&a, 0, sizeof(a));
    a.points = d_points; a.face = d_face; a.N = (int64_t)N; a.fnormal = d_face_normal; a.F = (int64_t)F;
    a.views = (const float4*)d_views; a.n_views = n_views; a.H = H; a.W = W; a.tol = depth_tol;
    a.rgb = d_rgb; a.weight = d_weight; a.view = d_view;
    for (int v = 0; v < n_views; ++v) {
        const float* P = h_poses + 16 * v;
        for (int r = 0; r < 3; ++r) {
            for (int c = 0; c < 3; ++c) a.rot[v][3 * r + c] = P[4 * r + c];
            a.cen[v][r] = P[4 * r + 3];
        }
    }
    if (N == 0) return PERF_OK;
#ifdef PERF_HOST_HARNESS
    (void)stream;
    for (int64_t i = 0; i < (int64_t)N; ++i) {
        PERF_CHECK_ARG(a.face[i] < (int32_t)F, "texel %lld: face %d of %llu", (long long)i, a.face[i], (unsigned long long)F);
        views_texel(a, i);
    }
#else
    views_kernel<<<(unsigned)((N + 127) / 128), 128, 0, (cudaStream_t)stream>>>(a);
    PERF_LAUNCH_CHECK();
#endif
    return PERF_OK;
}

#pragma GCC visibility pop
}
