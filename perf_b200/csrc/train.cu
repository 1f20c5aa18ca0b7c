// train.cu -- backward half of the fused training step: composite backward (thread = ray, marching
// back along the saved samples) and the grid-gradient scatter for ray-ordered samples.
#include <stdlib.h>
#include "common.cuh"

namespace perf {

struct CompBwdArgs {
    uint32_t S, seg; float near, far; uint64_t R; const float* toff;
    const float* jitter; const float* bg_noise;
    const float *sigma, *w, *T; const __half* rgb;
    const float *dist_acc;
    const float *g_rgb, *g_dist, *g_op, *g_dl, *dist_out, *op_out;
    float* out;
};

// dL/dw_i for the density phase:
//   distance_out = relu(D + c (1 - O)),  D = sum w m,  O = sum w,  c = 2 u - 1      (nerf_renderer.py:192)
//   distortion numerator DL = sum iv w^2 / 3 + 2 sum_i w_i (m_i Wx_i - WMx_i)        (SURVEY Appendix B)
//   dDL/dw_i = 2/3 iv_i w_i + 2 (m_i Wx_i - WMx_i) + 2 (WMsuf_i - m_i Wsuf_i)
// and dL/d(sigma_i dt_i) = (T_i - w_i) g_i - sum_{j>i} w_j g_j.
template <int PHASE>
__host__ __device__ __forceinline__ void composite_bwd_ray(const CompBwdArgs& a, uint64_t ray)
{
    const uint32_t S = a.S;
    const float step = fixed_s_step(a.near, a.far, S);
    const float jit = a.jitter ? a.jitter[ray] : 0.f;
    if constexpr (PHASE == PERF_PHASE_APP) {
        float gr = 0.f, gg = 0.f, gb = 0.f;
        if (a.g_rgb) { gr = a.g_rgb[3 * ray]; gg = a.g_rgb[3 * ray + 1]; gb = a.g_rgb[3 * ray + 2]; }
        const uint32_t kps = S / a.seg;
        for (uint32_t k = 0; k < S; ++k) {
            const uint64_t row = (uint64_t)k * a.R + ray;
            const float w = a.w[row] * (a.seg > 1 ? a.toff[(uint64_t)(k / kps) * a.R + ray] : 1.f);
            const uint2 c = *reinterpret_cast<const uint2*>(a.rgb + row * 4);
            const float2 c01 = unpack_half2(c.x), c2 = unpack_half2(c.y);
            // colours = sum w.detach() * rgb; rgb = sigmoid(z): dz = g * w * y (1 - y)
            a.out[row * 3 + 0] = gr * w * c01.x * (1.f - c01.x);
            a.out[row * 3 + 1] = gg * w * c01.y * (1.f - c01.y);
            a.out[row * 3 + 2] = gb * w * c2.x * (1.f - c2.x);
        }
    } else {
        const float O = a.op_out[ray], D = a.dist_acc[ray];
        float c = 0.f;
        if (a.bg_noise) c = a.bg_noise[4 * ray + 3] * 2.f - 1.f;
        const float mask = a.dist_out[ray] > 0.f ? 1.f : 0.f;
        const float gd = (a.g_dist ? a.g_dist[ray] : 0.f) * mask;
        const float gO = (a.g_op ? a.g_op[ray] : 0.f) - gd * c;
        const float gdl = a.g_dl ? a.g_dl[ray] : 0.f;
        float Wsuf = 0.f, WMsuf = 0.f, suf_wg = 0.f;
        const uint32_t kps = S / a.seg;
        for (uint32_t kk = S; kk-- > 0;) {
            const uint64_t row = (uint64_t)kk * a.R + ray;
            const float toff = a.seg > 1 ? a.toff[(uint64_t)(kk / kps) * a.R + ray] : 1.f;     // segment-local -> global
            const float w = a.w[row] * toff, T = a.T[row] * toff, sig = a.sigma[row];
            const float ts = fixed_s_t(a.near, step, kk, jit), te = fixed_s_t(a.near, step, kk + 1, jit);
            const float m = PERF_FADD_RN(ts, te) * 0.5f, dt = PERF_FSUB_RN(te, ts);
            const float Wx = O - Wsuf - w, WMx = D - WMsuf - w * m;
            const float ddl = (2.f / 3.f) * dt * w + 2.f * (m * Wx - WMx) + 2.f * (WMsuf - m * Wsuf);
            const float g = gd * m + gO + gdl * ddl;
            const float dsd = (T - w) * g - suf_wg;
            // trunc_exp backward (ngp_nerf.py:36-38): g * exp(clamp(raw, max=15)); sigma = exp(raw)
            a.out[row] = dsd * dt * fminf(sig, 3269017.3724721107f);
            suf_wg = fmaf(w, g, suf_wg); Wsuf += w; WMsuf = fmaf(w, m, WMsuf);
        }
    }
}

template <int PHASE>
__global__ void __launch_bounds__(128) composite_bwd_kernel(const CompBwdArgs a)
{
    const uint64_t ray = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (ray < a.R) composite_bwd_ray<PHASE>(a, ray);
}

// Chunk-parallel version of composite_bwd_ray (same formulas): an 8192-ray batch is only 64 CTAs of the kernel above,
// each thread walking 128 dependent samples.  Here a block is
// 32 consecutive rays (lanes: coalesced rows) x C chunks of S / C samples (warps); the suffix sums the backward scan
// needs (sum w, sum w m, sum w g over the LATER samples of the ray) are exchanged between the chunks through shared
// memory: pass 1 chunk sums of w and w m, pass 2 the backward walk inside the chunk, pass 3 the correction by the
// later chunks' sum w g.  Density phase only needs this; the colour phase has no dependence along the ray.
template <int PHASE, int C>
__global__ void __launch_bounds__(32 * C) composite_bwd_chunk_kernel(const CompBwdArgs a)
{
    const int rx = threadIdx.x, c = threadIdx.y;
    const uint64_t ray = (uint64_t)blockIdx.x * 32 + rx;
    const bool valid = ray < a.R;
    const uint32_t S = a.S, K = S / C, k_lo = c * K, k_hi = k_lo + K;
    const uint32_t kps = S / a.seg;
    const float step = __fdiv_rn(__fsub_rn(a.far, a.near), (float)S);     // fixed_s_step, kept inline: calling it changes this kernel's registers
    const float jit = (valid && a.jitter) ? a.jitter[ray] : 0.f;
    if constexpr (PHASE == PERF_PHASE_APP) {
        if (!valid) return;
        float gr = 0.f, gg = 0.f, gb = 0.f;
        if (a.g_rgb) { gr = a.g_rgb[3 * ray]; gg = a.g_rgb[3 * ray + 1]; gb = a.g_rgb[3 * ray + 2]; }
        for (uint32_t k = k_lo; k < k_hi; ++k) {
            const uint64_t row = (uint64_t)k * a.R + ray;
            const float w = a.w[row] * (a.seg > 1 ? a.toff[(uint64_t)(k / kps) * a.R + ray] : 1.f);
            const uint2 cc = *reinterpret_cast<const uint2*>(a.rgb + row * 4);
            const float2 c01 = unpack_half2(cc.x), c2 = unpack_half2(cc.y);
            a.out[row * 3 + 0] = gr * w * c01.x * (1.f - c01.x);
            a.out[row * 3 + 1] = gg * w * c01.y * (1.f - c01.y);
            a.out[row * 3 + 2] = gb * w * c2.x * (1.f - c2.x);
        }
    } else {
        __shared__ float sW[C][32], sWM[C][32], sWG[C][32];
        auto t_mid = [&](uint32_t k, float& m, float& dt) {
            const float ts = fixed_s_t(a.near, step, k, jit), te = fixed_s_t(a.near, step, k + 1, jit);
            m = __fadd_rn(ts, te) * 0.5f; dt = __fsub_rn(te, ts);
        };
        // pass 1: this chunk's sum w and sum w m
        float Wc = 0.f, WMc = 0.f;
        if (valid) {
            for (uint32_t k = k_lo; k < k_hi; ++k) {
                const uint64_t row = (uint64_t)k * a.R + ray;
                const float w = a.w[row] * (a.seg > 1 ? a.toff[(uint64_t)(k / kps) * a.R + ray] : 1.f);
                float m, dt; t_mid(k, m, dt);
                Wc += w; WMc = fmaf(w, m, WMc);
            }
        }
        sW[c][rx] = Wc; sWM[c][rx] = WMc;
        __syncthreads();
        float Wsuf = 0.f, WMsuf = 0.f;
        for (int cc = C - 1; cc > c; --cc) { Wsuf += sW[cc][rx]; WMsuf += sWM[cc][rx]; }
        // pass 2: backward walk inside the chunk
        float suf_wg = 0.f;
        float O = 0.f, D = 0.f, gd = 0.f, gO = 0.f, gdl = 0.f;
        if (valid) {
            O = a.op_out[ray]; D = a.dist_acc[ray];
            float cbg = 0.f;
            if (a.bg_noise) cbg = a.bg_noise[4 * ray + 3] * 2.f - 1.f;
            const float mask = a.dist_out[ray] > 0.f ? 1.f : 0.f;
            gd = (a.g_dist ? a.g_dist[ray] : 0.f) * mask;
            gO = (a.g_op ? a.g_op[ray] : 0.f) - gd * cbg;
            gdl = a.g_dl ? a.g_dl[ray] : 0.f;
            for (uint32_t kk = k_hi; kk-- > k_lo;) {
                const uint64_t row = (uint64_t)kk * a.R + ray;
                const float toff = a.seg > 1 ? a.toff[(uint64_t)(kk / kps) * a.R + ray] : 1.f;
                const float w = a.w[row] * toff, T = a.T[row] * toff, sig = a.sigma[row];
                float m, dt; t_mid(kk, m, dt);
                const float Wx = O - Wsuf - w, WMx = D - WMsuf - w * m;
                const float ddl = (2.f / 3.f) * dt * w + 2.f * (m * Wx - WMx) + 2.f * (WMsuf - m * Wsuf);
                const float g = gd * m + gO + gdl * ddl;
                const float dsd = (T - w) * g - suf_wg;
                a.out[row] = dsd * dt * fminf(sig, 3269017.3724721107f);
                suf_wg = fmaf(w, g, suf_wg); Wsuf += w; WMsuf = fmaf(w, m, WMsuf);
            }
        }
        sWG[c][rx] = suf_wg;
        __syncthreads();
        // pass 3: sum w g of the later chunks
        float off = 0.f;
        for (int cc = C - 1; cc > c; --cc) off += sWG[cc][rx];
        if (valid && off != 0.f) {
            for (uint32_t k = k_lo; k < k_hi; ++k) {
                const uint64_t row = (uint64_t)k * a.R + ray;
                float m, dt; t_mid(k, m, dt);
                a.out[row] -= off * dt * fminf(a.sigma[row], 3269017.3724721107f);
            }
        }
    }
}

// dh[n][j] = (sum_o dz[n][o] * wout[o][j]) * (h[n][j] > 0)   -- output layer backward + ReLU mask,
// one pass over the saved fp16 activations (8 columns per thread).
__global__ void __launch_bounds__(256)
mlp_bwd_out_kernel(const float* __restrict__ dz, int n_out, const __half* __restrict__ wout /*[n_out,64]*/,
                   const uint4* __restrict__ h /*[N,64] fp16*/, uint4* __restrict__ dh, uint64_t N)
{
    __shared__ float sw[16 * 64];
    for (int i = threadIdx.x; i < n_out * 64; i += blockDim.x) sw[i] = __half2float(wout[i]);
    __syncthreads();
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;       // one uint4 (8 halves)
    if (t >= N * 8) return;
    const uint64_t n = t >> 3; const int c0 = (int)(t & 7) * 8;
    float z[16];
    for (int o = 0; o < n_out; ++o) z[o] = dz[n * n_out + o];
    const uint4 hv = h[t];
    const uint32_t hw[4] = {hv.x, hv.y, hv.z, hv.w};
    uint32_t ow[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        const float2 hh = unpack_half2(hw[q]);
        float a = 0.f, b = 0.f;
        for (int o = 0; o < n_out; ++o) { a = fmaf(z[o], sw[o * 64 + c0 + 2 * q], a); b = fmaf(z[o], sw[o * 64 + c0 + 2 * q + 1], b); }
        ow[q] = pack_half2(hh.x > 0.f ? a : 0.f, hh.y > 0.f ? b : 0.f);
    }
    dh[t] = make_uint4(ow[0], ow[1], ow[2], ow[3]);
}

// dh[n][j] *= (h[n][j] > 0) in place (ReLU mask after a hidden-layer GEMM)
__global__ void __launch_bounds__(256)
relu_mask_kernel(uint4* __restrict__ dh, const uint4* __restrict__ h, uint64_t n16)
{
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n16) return;
    const uint4 hv = h[t]; uint4 d = dh[t];
    const uint32_t hw[4] = {hv.x, hv.y, hv.z, hv.w}; uint32_t dw[4] = {d.x, d.y, d.z, d.w};
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        const float2 hh = unpack_half2(hw[q]);
        if (!(hh.x > 0.f)) dw[q] &= 0xffff0000u;
        if (!(hh.y > 0.f)) dw[q] &= 0x0000ffffu;
    }
    dh[t] = make_uint4(dw[0], dw[1], dw[2], dw[3]);
}

// ---- grid-gradient scatter, rows sample-major, positions recomputed from the rays.
// Fine levels: one thread per (row, level), direct float2 atomics (lanes are neighbouring rays at the same
// sample index: at these resolutions they sit in different cells).  Coarse levels: see
// hashgrid_bwd_march_kernel below.
struct GridBwdRaysArgs {
    LevelTable lt;
    float aabb_min[3], aabb_ext[3];
    const float *rays_o, *rays_d, *jitter;
    uint64_t R; uint32_t S; float near, far;
    const float* dfeat; float2* dtable;
    uint64_t plane_rows;        // 0: dfeat is [N, 2 n_levels] rows; N > 0: level-major planes, plane l = float2 [N] (perf_mlp_bwd_scatter's output)
};

// One (row, level) of the fine-level scatter.  __host__ __device__ like the other per-thread bodies of this file:
// tests/host_harness.py runs them over host arrays (single thread, plain adds) against the oracle.
template <bool V4>
__host__ __device__ __forceinline__ void bwd_rays_row_level(const GridBwdRaysArgs& a, uint64_t row, int l)
{
    const uint64_t N = a.R * a.S;
    const bool live = row < N;
    float2 g = make_float2(0.f, 0.f);
    float x = 0.5f, y = 0.5f, z = 0.5f;
    if (live) {
        g = *reinterpret_cast<const float2*>(a.dfeat + row * (2 * a.lt.n_levels) + 2 * l);
        const uint64_t ray = row % a.R; const uint32_t k = (uint32_t)(row / a.R);
        const float step = fixed_s_step(a.near, a.far, a.S);
        const float jit = a.jitter ? a.jitter[ray] : 0.f;
        const float ts = fixed_s_t(a.near, step, k, jit), te = fixed_s_t(a.near, step, k + 1, jit);
        const float tsum = PERF_FADD_RN(ts, te);
        x = to_unit(sample_midpoint(a.rays_o[3 * ray], a.rays_d[3 * ray], tsum), a.aabb_min[0], a.aabb_ext[0]);
        y = to_unit(sample_midpoint(a.rays_o[3 * ray + 1], a.rays_d[3 * ray + 1], tsum), a.aabb_min[1], a.aabb_ext[1]);
        z = to_unit(sample_midpoint(a.rays_o[3 * ray + 2], a.rays_d[3 * ray + 2], tsum), a.aabb_min[2], a.aabb_ext[2]);
    }
    const bool active = live && (g.x != 0.f || g.y != 0.f);
    // level addressing with a dynamic level index (constant bank, uniform per block)
    const float scale = a.lt.scale[l];
    const uint32_t res = a.lt.res[l], size = a.lt.size[l], off = a.lt.offset[l];
    const bool hashed = (a.lt.hashed_mask >> l) & 1u, pow2 = (a.lt.pow2_mask >> l) & 1u;
    // common.cuh::cell_frame, kept inline: calling it changes the register allocation of hashgrid_bwd_rays_kernel<false>
    const float px = fmaf(scale, x, 0.5f), py = fmaf(scale, y, 0.5f), pz = fmaf(scale, z, 0.5f);
    const float fx = floorf(px), fy = floorf(py), fz = floorf(pz);
    const uint32_t gx = (uint32_t)(int)fx, gy = (uint32_t)(int)fy, gz = (uint32_t)(int)fz;
    float wx = px - fx, wy = py - fy, wz = pz - fz;
    if (a.lt.smoothstep) { wx = wx * wx * (3.f - 2.f * wx); wy = wy * wy * (3.f - 2.f * wy); wz = wz * wz * (3.f - 2.f * wz); }
    const float ox = 1.f - wx, oy = 1.f - wy, oz = 1.f - wz;
    float2 v[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const float w = active ? PERF_FMUL_RN(PERF_FMUL_RN((k & 1) ? wx : ox, (k & 2) ? wy : oy), (k & 4) ? wz : oz) : 0.f;
        v[k] = make_float2(w * g.x, w * g.y);
    }
    if (active) {
        uint32_t idx[8];
#pragma unroll
        for (int k = 0; k < 8; ++k)
            idx[k] = off + level_index(gx + (k & 1), gy + ((k >> 1) & 1), gz + ((k >> 2) & 1), hashed, pow2, res, size);
        scatter8<V4>(a.dtable, idx, v);
    }
}

template <bool V4>
__global__ void __launch_bounds__(256) hashgrid_bwd_rays_kernel(const __grid_constant__ GridBwdRaysArgs a)
{
    bwd_rays_row_level<V4>(a, (uint64_t)blockIdx.x * blockDim.x + threadIdx.x, (int)blockIdx.y);
}

// Coarse levels: one thread per (ray, level) walks the ray's S samples in order and keeps the 8
// corner sums of the CURRENT cell in registers; the 8 float2 atomics are issued only when the ray
// leaves the cell (consecutive samples of a ray stay ~17 / 12 / 8 / 5 ... samples in a level-0/1/2/3
// cell).  This divides the atomic count of the coarse levels -- the ones whose few addresses are hit
// by every ray near the camera -- by the run length.
template <bool V4>
__host__ __device__ __forceinline__ void bwd_march_ray_level(const GridBwdRaysArgs& a, uint64_t ray, int l, uint32_t piece, uint32_t n_pieces)
{
    // piece of the ray walked by this thread (more threads, shorter dependent loops; costs one extra flush per piece)
    const uint32_t k_per = (a.S + n_pieces - 1) / n_pieces;
    const uint32_t k_lo = piece * k_per, k_hi = a.S < k_lo + k_per ? a.S : k_lo + k_per;
    const float step = fixed_s_step(a.near, a.far, a.S);
    const float jit = a.jitter ? a.jitter[ray] : 0.f;
    const float ox = a.rays_o[3 * ray], oy = a.rays_o[3 * ray + 1], oz = a.rays_o[3 * ray + 2];
    const float dx = a.rays_d[3 * ray], dy = a.rays_d[3 * ray + 1], dz = a.rays_d[3 * ray + 2];
    const float scale = a.lt.scale[l];
    const uint32_t res = a.lt.res[l], size = a.lt.size[l], off = a.lt.offset[l];
    const bool hashed = (a.lt.hashed_mask >> l) & 1u, pow2 = (a.lt.pow2_mask >> l) & 1u;
    const uint32_t stride = 2 * a.lt.n_levels;
    uint32_t cx = 0xffffffffu, cy = 0xffffffffu, cz = 0xffffffffu;
    bool have = false;
    float2 acc[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) acc[k] = make_float2(0.f, 0.f);
    auto flush = [&]() {
        if constexpr (V4) {                                   // x-neighbour pairs as one 16-byte atomic (experimental, see perf_hashgrid_bwd_rays)
            uint32_t idx[8];
#pragma unroll
            for (int k = 0; k < 8; ++k) idx[k] = off + level_index(cx + (k & 1), cy + ((k >> 1) & 1), cz + ((k >> 2) & 1), hashed, pow2, res, size);
            scatter8<true>(a.dtable, idx, acc);
#pragma unroll
            for (int k = 0; k < 8; ++k) acc[k] = make_float2(0.f, 0.f);
        } else {
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                if (acc[k].x != 0.f || acc[k].y != 0.f) {
                    const uint32_t idx = off + level_index(cx + (k & 1), cy + ((k >> 1) & 1), cz + ((k >> 2) & 1), hashed, pow2, res, size);
                    grad_add2(a.dtable + idx, acc[k]);
                }
                acc[k] = make_float2(0.f, 0.f);
            }
        }
    };
#pragma unroll 2
    for (uint32_t ks = k_lo; ks < k_hi; ++ks) {
        const float2 g = a.plane_rows ? reinterpret_cast<const float2*>(a.dfeat)[(uint64_t)l * a.plane_rows + (uint64_t)ks * a.R + ray]
                                      : *reinterpret_cast<const float2*>(a.dfeat + ((uint64_t)ks * a.R + ray) * stride + 2 * l);
        if (g.x == 0.f && g.y == 0.f) continue;
        const float ts = fixed_s_t(a.near, step, ks, jit), te = fixed_s_t(a.near, step, ks + 1, jit);
        const float tsum = PERF_FADD_RN(ts, te);
        const float x = to_unit(sample_midpoint(ox, dx, tsum), a.aabb_min[0], a.aabb_ext[0]);
        const float y = to_unit(sample_midpoint(oy, dy, tsum), a.aabb_min[1], a.aabb_ext[1]);
        const float z = to_unit(sample_midpoint(oz, dz, tsum), a.aabb_min[2], a.aabb_ext[2]);
        // common.cuh::cell_frame, split around the cell test: calling it changes the registers of hashgrid_bwd_march_kernel
        const float px = fmaf(scale, x, 0.5f), py = fmaf(scale, y, 0.5f), pz = fmaf(scale, z, 0.5f);
        const float fx = floorf(px), fy = floorf(py), fz = floorf(pz);
        const uint32_t gx = (uint32_t)(int)fx, gy = (uint32_t)(int)fy, gz = (uint32_t)(int)fz;
        if (!have || gx != cx || gy != cy || gz != cz) {
            if (have) flush();
            cx = gx; cy = gy; cz = gz; have = true;
        }
        float wx = px - fx, wy = py - fy, wz = pz - fz;
        if (a.lt.smoothstep) { wx = wx * wx * (3.f - 2.f * wx); wy = wy * wy * (3.f - 2.f * wy); wz = wz * wz * (3.f - 2.f * wz); }
        const float oxw = 1.f - wx, oyw = 1.f - wy, ozw = 1.f - wz;
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const float w = PERF_FMUL_RN(PERF_FMUL_RN((k & 1) ? wx : oxw, (k & 2) ? wy : oyw), (k & 4) ? wz : ozw);
            acc[k].x = fmaf(w, g.x, acc[k].x); acc[k].y = fmaf(w, g.y, acc[k].y);
        }
    }
    if (have) flush();
}

template <bool V4>
__global__ void __launch_bounds__(128) hashgrid_bwd_march_kernel(const __grid_constant__ GridBwdRaysArgs a)
{
    const uint64_t ray = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (ray < a.R) bwd_march_ray_level<V4>(a, ray, (int)blockIdx.y, blockIdx.z, gridDim.z);
}

// Both scatter bodies in ONE launch: blocks of 256 threads, most of them fine-level blocks (thread = (row, level)), every
// (r+1)-th one a pair of coarse-level march blocks (thread = (ray, level, piece)).  Two separate launches -- even on two
// streams -- barely overlap: the fine kernel's blocks fill every SM and the latency-bound march blocks wait for them to
// retire (0.53 -> 0.50 ms); interleaved in one grid both kinds are resident together and the march kernel's latency hides
// behind the fine kernel's reductions.
struct GridBwdBothArgs {
    GridBwdRaysArgs a, b;        // a: all levels (coarse launch uses [0, n_agg)); b: the fine levels shifted down to index 0
    uint32_t n_agg, pieces, gx_march, gx_fine, n_fine_levels;
    uint32_t Bc, Bf, r;          // coarse 256-thread blocks, fine blocks, fine blocks per coarse block (interleave ratio)
};
template <bool V4>
__global__ void __launch_bounds__(256) hashgrid_bwd_both_kernel(const __grid_constant__ GridBwdBothArgs g)
{
    const uint32_t blk = blockIdx.x;
    uint32_t fine_idx, coarse_idx = 0xffffffffu;
    if (blk < g.Bc * (g.r + 1u)) {
        const uint32_t q = blk / (g.r + 1u), m = blk % (g.r + 1u);
        if (m < g.r) fine_idx = q * g.r + m; else { coarse_idx = q; fine_idx = 0xffffffffu; }
    } else {
        fine_idx = g.Bc * g.r + (blk - g.Bc * (g.r + 1u));
    }
    if (coarse_idx != 0xffffffffu) {
        const uint32_t mb = coarse_idx * 2u + (threadIdx.x >> 7);              // march block of 128 threads
        const uint32_t n_mb = g.gx_march * g.n_agg * g.pieces;
        if (mb < n_mb) {
            const uint32_t bx = mb % g.gx_march, level = (mb / g.gx_march) % g.n_agg, piece = mb / (g.gx_march * g.n_agg);
            const uint64_t ray = (uint64_t)bx * 128 + (threadIdx.x & 127);
            if (ray < g.a.R) bwd_march_ray_level<V4>(g.a, ray, (int)level, piece, g.pieces);
        }
    } else {
        const uint32_t bx = fine_idx % g.gx_fine, level = fine_idx / g.gx_fine;
        if (level < g.n_fine_levels) bwd_rays_row_level<V4>(g.b, (uint64_t)bx * 256 + threadIdx.x, (int)level);
    }
}

// ---- the scalar losses of a training step and their gradients w.r.t. the renderer outputs, ONE launch
// (nerf.py:208-238 density phase: smooth-L1 depth (beta 1e-2) + ramped distortion loss; nerf.py:281-287 colour phase:
// smooth-L1 colour (beta 5e-2)).  Replaces ~25 elementwise / reduction launches of the autograd graph per step.
struct LossArgs {
    uint64_t n;                  // elements of pred / gt (R or 3 R)
    uint64_t R;
    const float *pred, *gt; float beta, w_main;
    const float* dl; const float* ratio; const float* inv_n_rays; float w_dl;      // distortion loss (all null / 0 = off)
    float* loss;                 // [3]: total, main term (unweighted mean), distortion term (unweighted mean)
    float *g_pred, *g_dl;        // d total / d pred [n], d total / d dl [R]
};

__global__ void __launch_bounds__(1024) train_loss_kernel(const LossArgs a)
{
    __shared__ float red[2][32];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const float inv_n = 1.0f / (float)a.n;
    float s_main = 0.f, s_dl = 0.f;
    for (uint64_t i = tid; i < a.n; i += blockDim.x) {
        const float e = a.pred[i] - a.gt[i], ae = fabsf(e);
        float l, g;
        if (ae < a.beta) { l = 0.5f * e * e / a.beta; g = e / a.beta; }        // torch smooth_l1_loss
        else { l = ae - 0.5f * a.beta; g = e > 0.f ? 1.f : -1.f; }
        s_main += l;
        a.g_pred[i] = g * inv_n * a.w_main;
    }
    float k_dl = 0.f;
    if (a.dl) {
        k_dl = a.w_dl * (a.ratio ? a.ratio[0] : 1.f) * (a.inv_n_rays ? a.inv_n_rays[0] : 1.0f / (float)a.R);
        for (uint64_t r = tid; r < a.R; r += blockDim.x) { s_dl += a.dl[r]; a.g_dl[r] = k_dl; }
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) { s_main += __shfl_xor_sync(0xffffffffu, s_main, off); s_dl += __shfl_xor_sync(0xffffffffu, s_dl, off); }
    if (lane == 0) { red[0][warp] = s_main; red[1][warp] = s_dl; }
    __syncthreads();
    if (warp == 0) {
        float m = lane < (int)(blockDim.x >> 5) ? red[0][lane] : 0.f, d = lane < (int)(blockDim.x >> 5) ? red[1][lane] : 0.f;
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) { m += __shfl_xor_sync(0xffffffffu, m, off); d += __shfl_xor_sync(0xffffffffu, d, off); }
        if (lane == 0) {
            const float main_mean = m * inv_n;
            const float dl_term = a.dl ? d * (a.inv_n_rays ? a.inv_n_rays[0] : 1.0f / (float)a.R) : 0.f;       // flatten_eff_distloss
            a.loss[1] = main_mean; a.loss[2] = dl_term;
            a.loss[0] = a.w_main * main_mean + (a.dl ? a.w_dl * (a.ratio ? a.ratio[0] : 1.f) * dl_term : 0.f);
        }
    }
}

}  // namespace perf

using namespace perf;

extern "C" {
#pragma GCC visibility push(default)

static int setup_composite_bwd(int phase, uint32_t n_samples, uint32_t segments, float near, float far, uint64_t R,
                               const float* jitter, const float* bg_noise, const perf_train_buffers* buf,
                               const float* g_rgb, const float* g_distance, const float* g_opacity, const float* g_distloss,
                               const float* distance_out, const float* opacity_out, float* out, CompBwdArgs& a)
{
    PERF_CHECK_ARG(buf && out, "NULL pointer");
    PERF_CHECK_ARG(phase == PERF_PHASE_GEO || phase == PERF_PHASE_APP, "bad phase");
    PERF_CHECK_ARG(n_samples >= 1 && far > near, "bad sampling range");
    memset(&a, 0, sizeof(a));
    PERF_CHECK_ARG(segments >= 1 && n_samples % segments == 0 && (segments == 1 || buf->d_seg_trans), "bad segment count %u", segments);
    a.S = n_samples; a.seg = segments; a.toff = buf->d_seg_trans; a.near = near; a.far = far; a.R = R; a.jitter = jitter; a.bg_noise = bg_noise;
    a.sigma = buf->d_sigma; a.w = buf->d_weights; a.T = buf->d_trans; a.rgb = (const __half*)buf->d_rgb; a.dist_acc = buf->d_dist_acc;
    a.g_rgb = g_rgb; a.g_dist = g_distance; a.g_op = g_opacity; a.g_dl = g_distloss;
    a.dist_out = distance_out; a.op_out = opacity_out; a.out = out;
    if (R == 0) return PERF_OK;
    if (phase == PERF_PHASE_GEO) PERF_CHECK_ARG(a.sigma && a.w && a.T && a.dist_acc && a.dist_out && a.op_out, "density phase needs sigma/w/T/dist_acc and the forward outputs");
    else PERF_CHECK_ARG(a.w && a.rgb, "colour phase needs w and rgb");
    return PERF_OK;
}

int perf_train_backward_composite(int phase, uint32_t n_samples, uint32_t segments, float near, float far, uint64_t R,
                                  const float* d_jitter, const float* d_bg_noise, const perf_train_buffers* buf,
                                  const float* d_g_rgb, const float* d_g_distance, const float* d_g_opacity,
                                  const float* d_g_distloss, const float* d_distance_out, const float* d_opacity_out,
                                  float* d_out, void* stream)
{
    CompBwdArgs a;
    int rc = setup_composite_bwd(phase, n_samples, segments, near, far, R, d_jitter, d_bg_noise, buf, d_g_rgb, d_g_distance, d_g_opacity,
                                 d_g_distloss, d_distance_out, d_opacity_out, d_out, a);
    if (rc) return rc;
    if (R == 0) return PERF_OK;
    // chunk-parallel kernel when the ray-sequential one would leave the machine empty (PERF_B200_COMPBWD_CHUNKS=1: A/B)
    const char* env_c = getenv("PERF_B200_COMPBWD_CHUNKS");
    const bool chunked = !(env_c && env_c[0] == '1') && n_samples % 8 == 0 && n_samples >= 32 && (R + 127) / 128 < (uint64_t)num_sms() * 8;
    if (chunked) {
        const unsigned gridc = (unsigned)((R + 31) / 32);
        if (phase == PERF_PHASE_GEO) composite_bwd_chunk_kernel<PERF_PHASE_GEO, 8><<<gridc, dim3(32, 8), 0, (cudaStream_t)stream>>>(a);
        else composite_bwd_chunk_kernel<PERF_PHASE_APP, 8><<<gridc, dim3(32, 8), 0, (cudaStream_t)stream>>>(a);
    } else {
        const unsigned grid = (unsigned)((R + 127) / 128);
        if (phase == PERF_PHASE_GEO) composite_bwd_kernel<PERF_PHASE_GEO><<<grid, 128, 0, (cudaStream_t)stream>>>(a);
        else composite_bwd_kernel<PERF_PHASE_APP><<<grid, 128, 0, (cudaStream_t)stream>>>(a);
    }
    PERF_LAUNCH_CHECK();
    return PERF_OK;
}

#ifdef PERF_HOST_HARNESS
/* TEST HARNESS ONLY (never compiled into libperfb200.so): composite_bwd_ray over HOST arrays. */
int perf_host_train_backward_composite(int phase, uint32_t n_samples, uint32_t segments, float near, float far, uint64_t R,
                                       const float* h_jitter, const float* h_bg_noise, const perf_train_buffers* buf,
                                       const float* h_g_rgb, const float* h_g_distance, const float* h_g_opacity,
                                       const float* h_g_distloss, const float* h_distance_out, const float* h_opacity_out, float* h_out)
{
    CompBwdArgs a;
    int rc = setup_composite_bwd(phase, n_samples, segments, near, far, R, h_jitter, h_bg_noise, buf, h_g_rgb, h_g_distance, h_g_opacity,
                                 h_g_distloss, h_distance_out, h_opacity_out, h_out, a);
    if (rc) return rc;
    for (uint64_t ray = 0; ray < R; ++ray) { if (phase == PERF_PHASE_GEO) composite_bwd_ray<PERF_PHASE_GEO>(a, ray); else composite_bwd_ray<PERF_PHASE_APP>(a, ray); }
    return PERF_OK;
}
#endif

// argument blocks of the two scatter launches: `a` = all levels (the coarse launch uses levels [0, n_agg)),
// `b` = the remaining levels shifted down to index 0 (level table window + dfeat column window)
static int setup_bwd_rays(const perf_grid_cfg* cfg, const float* aabb6, const float* rays_o, const float* rays_d, const float* jitter,
                          uint64_t R, uint32_t n_samples, float near, float far, const float* dfeat, float* dtable,
                          GridBwdRaysArgs& a, GridBwdRaysArgs& b, uint32_t& n_agg)
{
    PERF_CHECK_ARG(aabb6 && rays_o && rays_d && dfeat && dtable, "NULL pointer");
    PERF_CHECK_ARG((uintptr_t)dtable % 8 == 0 && (uintptr_t)dfeat % 8 == 0, "misaligned dtable/dfeat");
    memset(&a, 0, sizeof(a));
    int rc = build_level_table(cfg, &a.lt, nullptr); if (rc) return rc;
    for (int i = 0; i < 3; ++i) { a.aabb_min[i] = aabb6[i]; a.aabb_ext[i] = aabb6[3 + i] - aabb6[i]; }
    a.rays_o = rays_o; a.rays_d = rays_d; a.jitter = jitter; a.R = R; a.S = n_samples; a.near = near; a.far = far;
    a.dfeat = dfeat; a.dtable = (float2*)dtable;
    // coarse levels: per-ray marching with register accumulation per cell; fine levels: direct atomics
    n_agg = a.lt.n_levels < 8 ? a.lt.n_levels : 8;
    b = a;
    for (uint32_t l = n_agg; l < a.lt.n_levels; ++l) {
        b.lt.scale[l - n_agg] = a.lt.scale[l]; b.lt.res[l - n_agg] = a.lt.res[l]; b.lt.size[l - n_agg] = a.lt.size[l]; b.lt.offset[l - n_agg] = a.lt.offset[l];
    }
    b.lt.hashed_mask = a.lt.hashed_mask >> n_agg; b.lt.pow2_mask = a.lt.pow2_mask >> n_agg;
    b.dfeat = a.dfeat + 2 * n_agg;                           // column window; row stride stays 2 * n_levels
    return PERF_OK;
}

int perf_hashgrid_bwd_rays(const perf_grid_cfg* cfg, const float* aabb6, const float* d_rays_o, const float* d_rays_d,
                           const float* d_jitter, uint64_t R, uint32_t n_samples, float near, float far,
                           const float* d_dfeat, float* d_dtable, void* stream)
{
    GridBwdRaysArgs a, b; uint32_t n_agg = 0;
    int rc = setup_bwd_rays(cfg, aabb6, d_rays_o, d_rays_d, d_jitter, R, n_samples, near, far, d_dfeat, d_dtable, a, b, n_agg); if (rc) return rc;
    const uint64_t N = R * n_samples;
    if (N == 0) return PERF_OK;
    // enough (ray, level, piece) threads to fill the machine; pieces of >= 16 samples
    unsigned pieces = 1;
    while (pieces < 8 && (uint64_t)R * n_agg * pieces < (uint64_t)num_sms() * 2048 && n_samples / (pieces * 2) >= 16) pieces *= 2;
    dim3 g_agg((unsigned)((R + 127) / 128), n_agg, pieces);
    {   // default: ONE launch with interleaved coarse / fine blocks (PERF_B200_SCATTER_MERGED=0: the two-launch path below)
        const char* env_m = getenv("PERF_B200_SCATTER_MERGED");
        const char* env_v4m = getenv("PERF_B200_SCATTER_V4");
        const bool v4m = !(env_v4m && env_v4m[0] == '0') && (uintptr_t)a.dtable % 16 == 0;
        if (!(env_m && env_m[0] == '0') && a.lt.n_levels > n_agg) {
            GridBwdBothArgs gb; gb.a = a; gb.b = b;
            gb.n_agg = n_agg; gb.pieces = pieces; gb.gx_march = g_agg.x; gb.gx_fine = (unsigned)((N + 255) / 256); gb.n_fine_levels = a.lt.n_levels - n_agg;
            const uint64_t n_mb = (uint64_t)g_agg.x * n_agg * pieces;
            gb.Bc = (uint32_t)((n_mb + 1) / 2); gb.Bf = gb.gx_fine * gb.n_fine_levels;
            gb.r = gb.Bc ? (gb.Bf / gb.Bc > 0 ? gb.Bf / gb.Bc : 1u) : 1u;
            if ((uint64_t)gb.Bc * gb.r > gb.Bf) gb.r = 1u;                      // more coarse than fine blocks: no interleave room
            if ((uint64_t)gb.Bc * gb.r <= gb.Bf) {
                const unsigned total = gb.Bc * (gb.r + 1u) + (gb.Bf - gb.Bc * gb.r);
                if (v4m) hashgrid_bwd_both_kernel<true><<<total, 256, 0, (cudaStream_t)stream>>>(gb);
                else hashgrid_bwd_both_kernel<false><<<total, 256, 0, (cudaStream_t)stream>>>(gb);
                PERF_LAUNCH_CHECK();
                return PERF_OK;
            }
        }
    }
    // The two launches touch disjoint halves of the gradient table and both sit on atomic latency, not bandwidth: run the
    // coarse one on a side stream (fork / join through events; capturable into a CUDA graph).  PERF_B200_SCATTER_OVERLAP=0
    // serialises them on the caller's stream as in round 1.
    cudaStream_t user = (cudaStream_t)stream, side = user;
    struct SideStream { cudaStream_t s; cudaEvent_t fork, join; };
    static thread_local SideStream s_sides[64] = {};                  // one per device, created on first use, never freed
    const char* env_ov = getenv("PERF_B200_SCATTER_OVERLAP");
    bool overlap = !(env_ov && env_ov[0] == '0') && a.lt.n_levels > n_agg;
    cudaEvent_t ev_join = nullptr;
    if (overlap) {
        int dev = 0; PERF_CUDA(cudaGetDevice(&dev));
        if (dev < 0 || dev >= 64) overlap = false;
        else {
            SideStream& ss = s_sides[dev];
            if (!ss.s) {
                PERF_CUDA(cudaStreamCreateWithFlags(&ss.s, cudaStreamNonBlocking));
                PERF_CUDA(cudaEventCreateWithFlags(&ss.fork, cudaEventDisableTiming));
                PERF_CUDA(cudaEventCreateWithFlags(&ss.join, cudaEventDisableTiming));
            }
            side = ss.s; ev_join = ss.join;
            PERF_CUDA(cudaEventRecord(ss.fork, user));
            PERF_CUDA(cudaStreamWaitEvent(side, ss.fork, 0));
        }
    }
    // the coarse flush uses the same 16-byte pair atomics: 0.586 -> 0.528 ms for both scatter launches of an 8192 x 128
    // step (tools/ab_scatter_v4.py); PERF_B200_SCATTER_V4_COARSE=0 restores the 8-byte flush
    const char* env_v4c = getenv("PERF_B200_SCATTER_V4_COARSE");
    if (!(env_v4c && env_v4c[0] == '0') && (uintptr_t)a.dtable % 16 == 0) hashgrid_bwd_march_kernel<true><<<g_agg, 128, 0, side>>>(a);
    else hashgrid_bwd_march_kernel<false><<<g_agg, 128, 0, side>>>(a);
    PERF_LAUNCH_CHECK();
    if (a.lt.n_levels > n_agg) {
        dim3 g_rest((unsigned)((N + 255) / 256), a.lt.n_levels - n_agg);
        // 16-byte vector atomics for x-neighbour pairs (REDG.E.ADD.F32x4): 0.659 -> 0.586 ms for the two scatter
        // launches of an 8192 x 128 step (tools/ab_scatter_v4.py); PERF_B200_SCATTER_V4=0 restores the 8-byte path
        const char* env_v4 = getenv("PERF_B200_SCATTER_V4");
        const bool want_v4 = !(env_v4 && env_v4[0] == '0');
        if (want_v4 && (uintptr_t)b.dtable % 16 == 0) hashgrid_bwd_rays_kernel<true><<<g_rest, 256, 0, user>>>(b);
        else hashgrid_bwd_rays_kernel<false><<<g_rest, 256, 0, user>>>(b);
        PERF_LAUNCH_CHECK();
    }
    if (overlap) {
        PERF_CUDA(cudaEventRecord(ev_join, side));
        PERF_CUDA(cudaStreamWaitEvent(user, ev_join, 0));
    }
    return PERF_OK;
}

/* The coarse levels [0, 8) only (run-merging march kernel): the companion of perf_mlp_bwd_scatter, whose epilogue has already
 * issued the fine levels' reductions.  d_dfeat: the eight level-major planes (float2 [N] each) that kernel wrote. */
int perf_hashgrid_bwd_rays_coarse(const perf_grid_cfg* cfg, const float* aabb6, const float* d_rays_o, const float* d_rays_d,
                                  const float* d_jitter, uint64_t R, uint32_t n_samples, float near, float far,
                                  const float* d_dfeat, float* d_dtable, void* stream)
{
    GridBwdRaysArgs a, b; uint32_t n_agg = 0;
    int rc = setup_bwd_rays(cfg, aabb6, d_rays_o, d_rays_d, d_jitter, R, n_samples, near, far, d_dfeat, d_dtable, a, b, n_agg); if (rc) return rc;
    if (R * (uint64_t)n_samples == 0) return PERF_OK;
    PERF_CHECK_SUP(a.lt.n_levels == 16 && n_agg == 8, "the fused scatter pair needs 16 levels (8 coarse planes)");
    a.plane_rows = R * (uint64_t)n_samples;
    unsigned pieces = 1;
    while (pieces < 8 && (uint64_t)R * n_agg * pieces < (uint64_t)num_sms() * 2048 && n_samples / (pieces * 2) >= 16) pieces *= 2;
    dim3 g_agg((unsigned)((R + 127) / 128), n_agg, pieces);
    if ((uintptr_t)a.dtable % 16 == 0) hashgrid_bwd_march_kernel<true><<<g_agg, 128, 0, (cudaStream_t)stream>>>(a);
    else hashgrid_bwd_march_kernel<false><<<g_agg, 128, 0, (cudaStream_t)stream>>>(a);
    PERF_LAUNCH_CHECK();
    return PERF_OK;
}

#ifdef PERF_HOST_HARNESS
/* TEST HARNESS ONLY (never compiled into libperfb200.so): both scatter bodies over HOST arrays, one thread;
 * `pieces` plays gridDim.z of the coarse launch, `v4` bit 0 / bit 1 select scatter8<true> for the fine / coarse levels. */
int perf_host_hashgrid_bwd_rays(const perf_grid_cfg* cfg, const float* aabb6, const float* h_rays_o, const float* h_rays_d,
                                const float* h_jitter, uint64_t R, uint32_t n_samples, float near, float far,
                                const float* h_dfeat, float* h_dtable, int v4, uint32_t pieces)
{
    GridBwdRaysArgs a, b; uint32_t n_agg = 0;
    int rc = setup_bwd_rays(cfg, aabb6, h_rays_o, h_rays_d, h_jitter, R, n_samples, near, far, h_dfeat, h_dtable, a, b, n_agg); if (rc) return rc;
    PERF_CHECK_ARG(pieces >= 1 && (!v4 || (uintptr_t)h_dtable % 16 == 0), "bad harness arguments");
    for (uint32_t l = 0; l < n_agg; ++l)
        for (uint32_t p = 0; p < pieces; ++p)
            for (uint64_t ray = 0; ray < R; ++ray) { if (v4 & 2) bwd_march_ray_level<true>(a, ray, (int)l, p, pieces); else bwd_march_ray_level<false>(a, ray, (int)l, p, pieces); }
    for (uint32_t l = 0; l + n_agg < a.lt.n_levels; ++l)
        for (uint64_t row = 0; row < R * n_samples; ++row) { if (v4 & 1) bwd_rays_row_level<true>(b, row, (int)l); else bwd_rays_row_level<false>(b, row, (int)l); }
    return PERF_OK;
}
#endif

int perf_train_loss(const float* d_pred, const float* d_gt, uint64_t n, uint64_t R, float beta, float w_main,
                    const float* d_distloss, const float* d_ratio, const float* d_inv_n_rays, float w_distloss,
                    float* d_loss3, float* d_g_pred, float* d_g_distloss, void* stream)
{
    PERF_CHECK_ARG(d_pred && d_gt && d_loss3 && d_g_pred, "NULL pointer");
    PERF_CHECK_ARG(n >= 1 && R >= 1 && beta > 0.f, "bad sizes / beta");
    PERF_CHECK_ARG(!d_distloss || d_g_distloss, "distortion loss needs d_g_distloss");
    LossArgs a; memset(&a, 0, sizeof(a));
    a.n = n; a.R = R; a.pred = d_pred; a.gt = d_gt; a.beta = beta; a.w_main = w_main;
    a.dl = d_distloss; a.ratio = d_ratio; a.inv_n_rays = d_inv_n_rays; a.w_dl = w_distloss;
    a.loss = d_loss3; a.g_pred = d_g_pred; a.g_dl = d_g_distloss;
    train_loss_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(a);
    PERF_LAUNCH_CHECK();
    return PERF_OK;
}

int perf_mlp_bwd_out(const float* d_dz, int n_out, const void* d_wout_half, const void* d_h, void* d_dh, uint64_t N, void* stream)
{
    PERF_CHECK_ARG(d_dz && d_wout_half && d_h && d_dh, "NULL pointer");
    PERF_CHECK_ARG(n_out >= 1 && n_out <= 16, "n_out=%d not in [1,16]", n_out);
    PERF_CHECK_ARG(((uintptr_t)d_h | (uintptr_t)d_dh) % 16 == 0, "misaligned activations");
    if (N == 0) return PERF_OK;
    mlp_bwd_out_kernel<<<(unsigned)((N * 8 + 255) / 256), 256, 0, (cudaStream_t)stream>>>(d_dz, n_out, (const __half*)d_wout_half, (const uint4*)d_h, (uint4*)d_dh, N);
    PERF_LAUNCH_CHECK();
    return PERF_OK;
}

int perf_relu_mask(void* d_dh, const void* d_h, uint64_t n_values, void* stream)
{
    PERF_CHECK_ARG(d_dh && d_h, "NULL pointer");
    PERF_CHECK_ARG(n_values % 8 == 0 && ((uintptr_t)d_h | (uintptr_t)d_dh) % 16 == 0, "n_values must be a multiple of 8 and buffers 16-byte aligned");
    if (n_values == 0) return PERF_OK;
    relu_mask_kernel<<<(unsigned)((n_values / 8 + 255) / 256), 256, 0, (cudaStream_t)stream>>>((uint4*)d_dh, (const uint4*)d_h, n_values / 8);
    PERF_LAUNCH_CHECK();
    return PERF_OK;
}

#pragma GCC visibility pop
}  // extern "C"
