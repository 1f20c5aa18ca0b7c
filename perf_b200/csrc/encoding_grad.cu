// encoding_grad.cu -- gradients of the hash-grid encode w.r.t. the INPUT positions, and their double
// backward (SURVEY.md §8(f) row 4).
//
// Replaces tiny-cuda-nn 1.7 (third-party, not vendored) `kernel_grid_backward_input`,
// `kernel_grid_backward_input_backward_grid`, `kernel_grid_backward_input_backward_dLdoutput` and
// `kernel_grid_backward_input_backward_input`, which the reference reaches through
// `tcnn.Encoding(... "interpolation": "Smoothstep")` and
// `torch.autograd.grad(distance, directions, create_graph=True)` in
// /root/reference/modules/geo_predictors/pano_joint_predictor.py:30-41,48-68 and
// /root/reference/modules/geo_predictors/pano_geo_refiner.py:19.
//
// Per level, with p = fract(scale*x + 0.5), s = p (Linear) or p^2(3-2p) (Smoothstep), omega_1 = s,
// omega_0 = 1-s and v_c the table entry of corner c:
//     y      = sum_c  prod_d omega_{c_d}(s_d) * v_c
//     dy/dx_d          = scale   * s'(p_d)          * A_d ,  A_d  = sum_{other two dims} omega*omega * (v_right - v_left)
//     d2y/dx_d^2       = scale^2 * s''(p_d)         * A_d
//     d2y/dx_d dx_e    = scale^2 * s'(p_d) s'(p_e)  * B_de,  B_de = sum_{third dim} omega * (v_11 - v_10 - v_01 + v_00)
// The table is the fp16 shadow (as in the forward); all arithmetic here is fp32 and the outputs are fp32.
// Oracle: autograd through oracle/hashgrid.py::encode_autograd.
//
// The per-sample bodies are __host__ __device__: compiled with -DPERF_HOST_HARNESS (tests only, a separate
// shared object built by tests/host_harness.py -- never part of libperfb200.so) two extra entry points run
// the SAME bodies over host arrays, so the arithmetic of this file is checked against the oracle on
// machines without a GPU.  The product library has no host path.
#include "grid_grad.cuh"

namespace perf {

__host__ __device__ __forceinline__ void load_corners(const __half2* __restrict__ table, const LevelFrame& f, float2 (&v)[8])
{
#pragma unroll
    for (int k = 0; k < 8; ++k) v[k] = __half22float2(table[f.idx[k]]);
}

__host__ __device__ __forceinline__ void accumulate(float* p, float v)
{
#ifdef __CUDA_ARCH__
    atomicAdd(p, v);
#else
    *p += v;                       // host harness: single thread
#endif
}

// ---- dL/dx = sum_levels sum_f dL/dy_f * dy_f/dx : one sample, all levels.
__host__ __device__ __forceinline__ void bwd_input_sample(const LevelTable& lt, const __half2* __restrict__ table,
                                                          const float* __restrict__ x01, const float* __restrict__ dfeat,
                                                          uint64_t i, float* __restrict__ dx)
{
    const float x = x01[3 * i], y = x01[3 * i + 1], z = x01[3 * i + 2];
    const float2* g = reinterpret_cast<const float2*>(dfeat) + i * lt.n_levels;
    float acc[3] = {0.f, 0.f, 0.f};
    for (int l = 0; l < (int)lt.n_levels; ++l) {
        LevelFrame f; level_frame(lt, l, x, y, z, f);
        float2 v[8]; load_corners(table, f, v);
        const float2 gl = g[l];
        const float2 a0 = diff_along<0>(f, v), a1 = diff_along<1>(f, v), a2 = diff_along<2>(f, v);
        acc[0] = fmaf(f.scale * f.ds[0], fmaf(gl.x, a0.x, gl.y * a0.y), acc[0]);
        acc[1] = fmaf(f.scale * f.ds[1], fmaf(gl.x, a1.x, gl.y * a1.y), acc[1]);
        acc[2] = fmaf(f.scale * f.ds[2], fmaf(gl.x, a2.x, gl.y * a2.y), acc[2]);
    }
    dx[3 * i] = acc[0]; dx[3 * i + 1] = acc[1]; dx[3 * i + 2] = acc[2];
}

__global__ void __launch_bounds__(256)
encoding_bwd_input_kernel(LevelTable lt, const __half2* __restrict__ table, const float* __restrict__ x01,
                          const float* __restrict__ dfeat, uint64_t N, float* __restrict__ dx)
{
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < N) bwd_input_sample(lt, table, x01, dfeat, i, dx);
}

// ---- double backward of dL/dx.  With u = d(loss2)/d(dL/dx) [N,3] and g = dL/dy [N,2L]:
//   ddfeat[i, l, f] = sum_d u_d * dy_f/dx_d                          (gradient w.r.t. g)
//   dtable[c]      += (sum_d +-u_d * scale s'(p_d) * omega*omega) * g  (gradient w.r.t. the table)
//   dx2[i, e]      += sum_d u_d * sum_f g_f * d2y_f/dx_d dx_e          (gradient w.r.t. x)
// One thread per (sample, level): blockIdx.y = level.  dtable / dx2 are accumulated with atomics and
// must be zeroed by the caller; any of the three outputs may be NULL.
__host__ __device__ __forceinline__ void bwd_bwd_input_sample_level(
    const LevelTable& lt, const __half2* __restrict__ table, const float* __restrict__ x01, const float* __restrict__ dfeat,
    const float* __restrict__ ddx, uint64_t i, int l, float* __restrict__ ddfeat, float2* __restrict__ dtable, float* __restrict__ dx2)
{
    LevelFrame f; level_frame(lt, l, x01[3 * i], x01[3 * i + 1], x01[3 * i + 2], f);
    const float u[3] = {ddx[3 * i], ddx[3 * i + 1], ddx[3 * i + 2]};
    const float2 g = reinterpret_cast<const float2*>(dfeat)[i * lt.n_levels + l];
    const float j[3] = {f.scale * f.ds[0], f.scale * f.ds[1], f.scale * f.ds[2]};      // d s_d / d x_d

    if (dtable) {
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            // d/dv_k of sum_d u_d dy/dx_d: corner k is "right" along d when bit d is set
            float c = 0.f;
#pragma unroll
            for (int d = 0; d < 3; ++d) {
                const int e = (d + 1) % 3, h = (d + 2) % 3;
                const float w = (((k >> e) & 1) ? f.s[e] : 1.0f - f.s[e]) * (((k >> h) & 1) ? f.s[h] : 1.0f - f.s[h]);
                const float t = u[d] * j[d] * w;
                c += ((k >> d) & 1) ? t : -t;
            }
            if (c != 0.f) {
                accumulate(&dtable[f.idx[k]].x, c * g.x);
                accumulate(&dtable[f.idx[k]].y, c * g.y);
            }
        }
    }
    if (!ddfeat && !dx2) return;
    float2 v[8]; load_corners(table, f, v);
    const float2 a0 = diff_along<0>(f, v), a1 = diff_along<1>(f, v), a2 = diff_along<2>(f, v);
    if (ddfeat) {
        float2 r;
        r.x = u[0] * j[0] * a0.x + u[1] * j[1] * a1.x + u[2] * j[2] * a2.x;
        r.y = u[0] * j[0] * a0.y + u[1] * j[1] * a1.y + u[2] * j[2] * a2.y;
        reinterpret_cast<float2*>(ddfeat)[i * lt.n_levels + l] = r;
    }
    if (dx2) {
        const float2 b01 = diff_cross<0, 1>(f, v), b02 = diff_cross<0, 2>(f, v), b12 = diff_cross<1, 2>(f, v);
        const float ga[3]  = {g.x * a0.x + g.y * a0.y, g.x * a1.x + g.y * a1.y, g.x * a2.x + g.y * a2.y};
        const float gb01 = g.x * b01.x + g.y * b01.y, gb02 = g.x * b02.x + g.y * b02.y, gb12 = g.x * b12.x + g.y * b12.y;
        const float s2 = f.scale * f.scale;
        // Hessian of (g . y) w.r.t. x, contracted with u
        const float h00 = s2 * f.dds[0] * ga[0], h11 = s2 * f.dds[1] * ga[1], h22 = s2 * f.dds[2] * ga[2];
        const float h01 = j[0] * j[1] * gb01, h02 = j[0] * j[2] * gb02, h12 = j[1] * j[2] * gb12;
        accumulate(&dx2[3 * i],     u[0] * h00 + u[1] * h01 + u[2] * h02);
        accumulate(&dx2[3 * i + 1], u[0] * h01 + u[1] * h11 + u[2] * h12);
        accumulate(&dx2[3 * i + 2], u[0] * h02 + u[1] * h12 + u[2] * h22);
    }
}

__global__ void __launch_bounds__(256)
encoding_bwd_bwd_input_kernel(LevelTable lt, const __half2* __restrict__ table, const float* __restrict__ x01,
                              const float* __restrict__ dfeat, const float* __restrict__ ddx, uint64_t N,
                              float* __restrict__ ddfeat, float2* __restrict__ dtable, float* __restrict__ dx2)
{
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < N) bwd_bwd_input_sample_level(lt, table, x01, dfeat, ddx, i, (int)blockIdx.y, ddfeat, dtable, dx2);
}

}  // namespace perf

using namespace perf;
static inline unsigned blocks_for(uint64_t n, unsigned per) { return (unsigned)((n + per - 1) / per); }
#define S(stream) ((cudaStream_t)(stream))

extern "C" {
#pragma GCC visibility push(default)

int perf_hashgrid_bwd_input(const perf_grid_cfg* cfg, const void* d_table_half, const float* d_x01,
                                     const float* d_dfeat, uint64_t N, float* d_dx, void* stream)
{
    PERF_CHECK_ARG(d_table_half && d_x01 && d_dfeat && d_dx, "NULL pointer");
    LevelTable lt; int rc = build_level_table(cfg, &lt, nullptr); if (rc) return rc;
    PERF_CHECK_ARG((uintptr_t)d_table_half % 4 == 0 && (uintptr_t)d_dfeat % 8 == 0, "misaligned table/dfeat");
    if (N == 0) return PERF_OK;
    encoding_bwd_input_kernel<<<blocks_for(N, 256), 256, 0, S(stream)>>>(lt, (const __half2*)d_table_half, d_x01, d_dfeat, N, d_dx);
    PERF_LAUNCH_CHECK();
    return PERF_OK;
}

int perf_hashgrid_bwd_bwd_input(const perf_grid_cfg* cfg, const void* d_table_half, const float* d_x01,
                                         const float* d_dfeat, const float* d_ddx, uint64_t N,
                                         float* d_ddfeat, float* d_dtable, float* d_dx2, void* stream)
{
    PERF_CHECK_ARG(d_table_half && d_x01 && d_dfeat && d_ddx, "NULL pointer");
    PERF_CHECK_ARG(d_ddfeat || d_dtable || d_dx2, "no output requested");
    LevelTable lt; int rc = build_level_table(cfg, &lt, nullptr); if (rc) return rc;
    PERF_CHECK_ARG((uintptr_t)d_table_half % 4 == 0 && (uintptr_t)d_dfeat % 8 == 0 && (uintptr_t)d_ddfeat % 8 == 0 &&
                   (uintptr_t)d_dtable % 8 == 0, "misaligned table/dfeat/ddfeat/dtable");
    if (N == 0) return PERF_OK;
    encoding_bwd_bwd_input_kernel<<<dim3(blocks_for(N, 256), lt.n_levels), 256, 0, S(stream)>>>(
        lt, (const __half2*)d_table_half, d_x01, d_dfeat, d_ddx, N, d_ddfeat, (float2*)d_dtable, d_dx2);
    PERF_LAUNCH_CHECK();
    return PERF_OK;
}

#ifdef PERF_HOST_HARNESS
/* TEST HARNESS ONLY (not compiled into libperfb200.so): the bodies above over HOST arrays, one thread. */
int perf_host_hashgrid_bwd_input(const perf_grid_cfg* cfg, const void* h_table_half, const float* h_x01,
                                 const float* h_dfeat, uint64_t N, float* h_dx)
{
    LevelTable lt; int rc = build_level_table(cfg, &lt, nullptr); if (rc) return rc;
    for (uint64_t i = 0; i < N; ++i) bwd_input_sample(lt, (const __half2*)h_table_half, h_x01, h_dfeat, i, h_dx);
    return PERF_OK;
}

int perf_host_hashgrid_bwd_bwd_input(const perf_grid_cfg* cfg, const void* h_table_half, const float* h_x01,
                                     const float* h_dfeat, const float* h_ddx, uint64_t N,
                                     float* h_ddfeat, float* h_dtable, float* h_dx2)
{
    LevelTable lt; int rc = build_level_table(cfg, &lt, nullptr); if (rc) return rc;
    for (uint64_t i = 0; i < N; ++i)
        for (int l = 0; l < (int)lt.n_levels; ++l)
            bwd_bwd_input_sample_level(lt, (const __half2*)h_table_half, h_x01, h_dfeat, h_ddx, i, l, h_ddfeat, (float2*)h_dtable, h_dx2);
    return PERF_OK;
}
#endif

#pragma GCC visibility pop
}  // extern "C"
