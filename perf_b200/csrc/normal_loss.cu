// normal_loss.cu -- normal-consistency loss of the density phase (MonoSDF's L1 + angular normal loss on PeRF's supervision
// normals): the training-time sample normals, the ray normal N_r = sum_i sg(w_i) n_i, the loss and its gradient, and the
// second-order backward of the normals into W1, w_out and the hash table.  Definition: include/perfb200.h ("normal-consistency
// loss"), DESIGN §4.
//
// Per sample i at normalised position x01 (h1 = the fp16 layer-1 activation the training forward saved, m = [h1 > 0]):
//     g      = W1^T (m . w_out)                                   (32-vector, fp16 weights as fp32)
//     grad01 = sum_levels level_input_grad(g)                     (grid_grad.cuh, fp16 geo table)
//     n      = -(grad01 / ext) / |grad01 / ext|,   r = 1 / |grad01 / ext|
// Backward with G_r = dL/dN_r:  u = -(I - n n^T)(w_i G_r) r,  v = u / ext  (= dL/d grad01), and per level l, feature f
//     dg_{l,f}   = sum_d v_d scale s'(p_d) A_{d,l,f}                (encoding_grad.cu::bwd_bwd_input_sample_level, ddfeat)
//     dtable_c  += g_{l,f} sum_d +-v_d scale s'(p_d) omega omega     (same function, dtable)
//     P         += m (x) dg   (64 x 32),   dW1 = diag(w_out) P,   dw_out_j = sum_k W1_jk P_jk.
// The per-sample arithmetic is __host__ __device__: tests/host_harness.py builds this file with -DPERF_HOST_HARNESS and runs the
// same bodies over host arrays against tests/normal_loss_oracle.py.  The product library has no host path.
#include "grid_grad.cuh"

namespace perf {

constexpr int NL_LEVELS = 16, NL_HIDDEN = 64, NL_IN = 32;
constexpr int NL_THREADS = 256;

struct NlArgs {
    LevelTable lt;
    const __half2* table;                 // fp16 geo grid [n_entries] (feature pairs)
    const __half* w1;                     // fp16 W1 [64][32] (row j = hidden unit)
    const __half* wout;                   // fp16 output row 0 [64]
    float aabb_min[3], aabb_ext[3];
    uint64_t R, N;
    // packed layout (x01 != null)
    const float* x01; const int64_t* offsets; const int64_t* ray_indices; const int64_t* n_dev;
    // fixed-S layout (x01 == null): rows k * R + ray
    const float *rays_o, *rays_d, *jitter; uint32_t S, seg; float near, far; const float* seg_trans;
    // per-sample saves of the training forward
    const __half* h1; const float *w, *T;
    // normals (forward outputs, backward inputs)
    float* nrm; float* rinv; float* ray_nrm;
    // backward
    const float* g_ray; float* dmlp; float2* dtable;
};

// The sample's weight and transmittance along its whole ray (fixed-S: segment-local values times the segment's start T) and its ray.
__host__ __device__ __forceinline__ float nl_weight(const NlArgs& a, uint64_t i, float& T, uint64_t& ray)
{
    if (a.x01) {
        ray = a.ray_indices ? (uint64_t)a.ray_indices[i] : 0;
        T = a.T[i];
        return a.w[i];
    }
    ray = i % a.R;
    const uint32_t k = (uint32_t)(i / a.R);
    const float toff = a.seg > 1 ? a.seg_trans[(uint64_t)(k / (a.S / a.seg)) * a.R + ray] : 1.f;
    T = a.T[i] * toff;
    return a.w[i] * toff;
}

// Normalised position of sample i: the packed forward's saved x01, or the fixed-S position recomputed from the ray bit for bit
// as hashgrid_bwd_rays does (train.cu::bwd_rays_row_level).  Returns the selector.
__host__ __device__ __forceinline__ bool nl_position(const NlArgs& a, uint64_t i, float (&x)[3])
{
    if (a.x01) {
        x[0] = a.x01[3 * i]; x[1] = a.x01[3 * i + 1]; x[2] = a.x01[3 * i + 2];
    } else {
        const uint64_t ray = i % a.R; const uint32_t k = (uint32_t)(i / a.R);
        const float step = fixed_s_step(a.near, a.far, a.S);
        const float jit = a.jitter ? a.jitter[ray] : 0.f;
        const float tsum = PERF_FADD_RN(fixed_s_t(a.near, step, k, jit), fixed_s_t(a.near, step, k + 1, jit));
#pragma unroll
        for (int d = 0; d < 3; ++d) x[d] = to_unit(sample_midpoint(a.rays_o[3 * ray + d], a.rays_d[3 * ray + d], tsum), a.aabb_min[d], a.aabb_ext[d]);
    }
    return x[0] > 0.f && x[0] < 1.f && x[1] > 0.f && x[1] < 1.f && x[2] > 0.f && x[2] < 1.f;
}

// m = [h1 > 0] (64 bits) and g = W1^T (m . w_out).  w1 [64*32] / wout [64] fp32 (shared memory on the device).
__host__ __device__ __forceinline__ void nl_g(const float* __restrict__ w1, const float* __restrict__ wout, const __half* __restrict__ h1row,
                                              float (&g)[NL_IN], uint32_t (&m)[2])
{
    m[0] = m[1] = 0u;
#pragma unroll
    for (int q = 0; q < 8; ++q) {
        const uint4 hv = *reinterpret_cast<const uint4*>(h1row + 8 * q);
        const uint32_t hw[4] = {hv.x, hv.y, hv.z, hv.w};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const float2 hh = unpack_half2(hw[e]);
            const int j = 8 * q + 2 * e;
            if (hh.x > 0.f) m[j >> 5] |= 1u << (j & 31);
            if (hh.y > 0.f) m[(j + 1) >> 5] |= 1u << ((j + 1) & 31);
        }
    }
#pragma unroll
    for (int k = 0; k < NL_IN; ++k) g[k] = 0.f;
#pragma unroll 4
    for (int j = 0; j < NL_HIDDEN; ++j) {
        const float mw = ((m[j >> 5] >> (j & 31)) & 1u) ? wout[j] : 0.f;
#pragma unroll
        for (int k = 0; k < NL_IN; ++k) g[k] = fmaf(w1[j * NL_IN + k], mw, g[k]);
    }
}

__host__ __device__ __forceinline__ void nl_corners(const __half2* __restrict__ table, const LevelFrame& f, float2 (&v)[8])
{
#pragma unroll
    for (int k = 0; k < 8; ++k) v[k] = __half22float2(table[f.idx[k]]);
}

// n and r = 1 / |grad| of one sample from its position and g (the eval normals' arithmetic: render.cu::sample_normal).
__host__ __device__ __forceinline__ void nl_normal(const NlArgs& a, const float (&x)[3], const float (&g)[NL_IN], float (&n)[3], float& r)
{
    float acc[3] = {0.f, 0.f, 0.f};
#pragma unroll 1
    for (int l = 0; l < NL_LEVELS; ++l) {
        LevelFrame f; level_frame(a.lt, l, x[0], x[1], x[2], f);
        float2 v[8]; nl_corners(a.table, f, v);
        float2 gl;
        // dynamic level index into g: select from the register array instead of spilling it to local memory
        gl.x = 0.f; gl.y = 0.f;
#pragma unroll
        for (int q = 0; q < NL_LEVELS; ++q) if (q == l) { gl.x = g[2 * q]; gl.y = g[2 * q + 1]; }
        level_input_grad(f, v, gl, acc);
    }
    const float gx = acc[0] / a.aabb_ext[0], gy = acc[1] / a.aabb_ext[1], gz = acc[2] / a.aabb_ext[2];
    const float nn = sqrtf(gx * gx + gy * gy + gz * gz);
    r = nn > 0.f ? 1.f / nn : 0.f;
    n[0] = -gx * r; n[1] = -gy * r; n[2] = -gz * r;
}

// Forward of one sample: n_i and r_i, both 0 for a sample that does not reach its ray normal (w = 0, T = 0 -- a dropped sample --,
// selector false, or |grad| = 0).  w1 / wout: fp32 copies of the fp16 weights.
__host__ __device__ __forceinline__ void nl_fwd_sample(const NlArgs& a, const float* w1, const float* wout, uint64_t i)
{
    float T; uint64_t ray;
    const float w = nl_weight(a, i, T, ray);
    float n[3] = {0.f, 0.f, 0.f}, r = 0.f;
    float x[3];
    if (w != 0.f && T != 0.f && nl_position(a, i, x)) {
        float g[NL_IN]; uint32_t m[2];
        nl_g(w1, wout, a.h1 + i * NL_HIDDEN, g, m);
        nl_normal(a, x, g, n, r);
    }
    a.nrm[3 * i] = n[0]; a.nrm[3 * i + 1] = n[1]; a.nrm[3 * i + 2] = n[2];
    a.rinv[i] = r;
}

// Fixed-S ray normal, thread = ray: N_r = sum_k w n over the S rows in order.
__host__ __device__ __forceinline__ void nl_ray_sum_fixed(const NlArgs& a, uint64_t ray)
{
    float s0 = 0.f, s1 = 0.f, s2 = 0.f;
    for (uint32_t k = 0; k < a.S; ++k) {
        const uint64_t i = (uint64_t)k * a.R + ray;
        float T; uint64_t rr;
        const float w = nl_weight(a, i, T, rr);
        if (a.rinv[i] == 0.f) continue;
        s0 = fmaf(w, a.nrm[3 * i], s0); s1 = fmaf(w, a.nrm[3 * i + 1], s1); s2 = fmaf(w, a.nrm[3 * i + 2], s2);
    }
    a.ray_nrm[3 * ray] = s0; a.ray_nrm[3 * ray + 1] = s1; a.ray_nrm[3 * ray + 2] = s2;
}

// The loss of one ray (MonoSDF: L1 + angular on the normalised rendered normal): returns validity, l and dl/dN.
__host__ __device__ __forceinline__ bool nl_loss_ray(const float (&N)[3], const float (&gt)[3], float& l, float (&dl)[3])
{
    const float gn = sqrtf(gt[0] * gt[0] + gt[1] * gt[1] + gt[2] * gt[2]);
    const float Nn = sqrtf(N[0] * N[0] + N[1] * N[1] + N[2] * N[2]);
    l = 0.f; dl[0] = dl[1] = dl[2] = 0.f;
    if (!(gn > 0.5f && Nn > 1e-6f)) return false;
    float gh[3], nh[3], s[3];
#pragma unroll
    for (int d = 0; d < 3; ++d) { gh[d] = gt[d] / gn; nh[d] = N[d] / Nn; }
    float dot = 0.f, l1 = 0.f, na = 0.f;
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        const float e = nh[d] - gh[d];
        l1 += fabsf(e);
        dot = fmaf(nh[d], gh[d], dot);
        s[d] = (e > 0.f ? 1.f : (e < 0.f ? -1.f : 0.f)) - gh[d];          // dl/d(N^) with sign(0) = 0
        na = fmaf(nh[d], s[d], na);
    }
    l = l1 + (1.f - dot);
#pragma unroll
    for (int d = 0; d < 3; ++d) dl[d] = (s[d] - nh[d] * na) / Nn;          // (I - N^ N^T) s / |N|
    return true;
}

// Backward of one sample: v = dL/d grad01 (written to v_out when non-null), then per level dg (written to dg_out [32] when
// non-null) and the table atomics.  Returns false (and touches nothing) when the sample issues nothing.
__host__ __device__ __forceinline__ bool nl_bwd_sample(const NlArgs& a, const float* w1, const float* wout, uint64_t i,
                                                       float (&dg)[NL_IN], uint32_t (&m)[2], float* v_out)
{
    float T; uint64_t ray;
    const float w = nl_weight(a, i, T, ray);
    const float r = a.rinv[i];
    if (w == 0.f || T == 0.f || r == 0.f) return false;
    const float G[3] = {a.g_ray[3 * ray] * w, a.g_ray[3 * ray + 1] * w, a.g_ray[3 * ray + 2] * w};
    if (G[0] == 0.f && G[1] == 0.f && G[2] == 0.f) return false;
    float x[3];
    nl_position(a, i, x);
    float g[NL_IN];
    nl_g(w1, wout, a.h1 + i * NL_HIDDEN, g, m);
    const float n[3] = {a.nrm[3 * i], a.nrm[3 * i + 1], a.nrm[3 * i + 2]};
    const float nG = n[0] * G[0] + n[1] * G[1] + n[2] * G[2];
    float v[3];
#pragma unroll
    for (int d = 0; d < 3; ++d) v[d] = -(G[d] - n[d] * nG) * r / a.aabb_ext[d];
    if (v_out) { v_out[0] = v[0]; v_out[1] = v[1]; v_out[2] = v[2]; }
#pragma unroll 1
    for (int l = 0; l < NL_LEVELS; ++l) {
        LevelFrame f; level_frame(a.lt, l, x[0], x[1], x[2], f);
        const float j[3] = {f.scale * f.ds[0], f.scale * f.ds[1], f.scale * f.ds[2]};      // d s_d / d x_d
        float2 gl = make_float2(0.f, 0.f);
#pragma unroll
        for (int q = 0; q < NL_LEVELS; ++q) if (q == l) { gl.x = g[2 * q]; gl.y = g[2 * q + 1]; }
        // dtable: d/dv_k of sum_d v_d dy/dx_d, corner k "right" along d when bit d is set
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            float c = 0.f;
#pragma unroll
            for (int d = 0; d < 3; ++d) {
                const int e = (d + 1) % 3, h = (d + 2) % 3;
                const float om = (((k >> e) & 1) ? f.s[e] : 1.0f - f.s[e]) * (((k >> h) & 1) ? f.s[h] : 1.0f - f.s[h]);
                const float t = v[d] * j[d] * om;
                c += ((k >> d) & 1) ? t : -t;
            }
            if (c != 0.f) grad_add2(a.dtable + f.idx[k], make_float2(c * gl.x, c * gl.y));
        }
        // dg: sum_d v_d dy_f/dx_d
        float2 cv[8]; nl_corners(a.table, f, cv);
        const float2 a0 = diff_along<0>(f, cv), a1 = diff_along<1>(f, cv), a2 = diff_along<2>(f, cv);
        const float rx = v[0] * j[0] * a0.x + v[1] * j[1] * a1.x + v[2] * j[2] * a2.x;
        const float ry = v[0] * j[0] * a0.y + v[1] * j[1] * a1.y + v[2] * j[2] * a2.y;
#pragma unroll
        for (int q = 0; q < NL_LEVELS; ++q) if (q == l) { dg[2 * q] = rx; dg[2 * q + 1] = ry; }
    }
    return true;
}

// dW1 = diag(w_out) P, dw_out_j = sum_k W1_jk P_jk for rows j, columns [k0, k0 + K) of P: the gradient of the MLP weights in the
// flat parameter layout (W1 at 0, output row 0 at 64 * 32).  Returns this piece's share of dw_out_j (the caller adds the pieces).
template <int K>
__host__ __device__ __forceinline__ float nl_flush_row(const float* w1, const float* wout, int j, int k0, const float (&P)[K], float* dmlp)
{
    float dwo = 0.f;
#pragma unroll
    for (int kk = 0; kk < K; ++kk) {
        const float dw = wout[j] * P[kk];
        if (dw != 0.f) {
#ifdef __CUDA_ARCH__
            atomicAdd(dmlp + j * NL_IN + k0 + kk, dw);
#else
            dmlp[j * NL_IN + k0 + kk] += dw;
#endif
        }
        dwo = fmaf(w1[j * NL_IN + k0 + kk], P[kk], dwo);
    }
    return dwo;
}

// ---------------------------------------------------------------- kernels
__device__ __forceinline__ uint64_t nl_live(const NlArgs& a) { return a.n_dev ? (uint64_t)min((int64_t)a.N, max(*a.n_dev, (int64_t)0)) : a.N; }

__device__ __forceinline__ void nl_stage_weights(const NlArgs& a, float* s_w1, float* s_wo)
{
    for (int t = threadIdx.x; t < NL_HIDDEN * NL_IN; t += blockDim.x) s_w1[t] = __half2float(a.w1[t]);
    for (int t = threadIdx.x; t < NL_HIDDEN; t += blockDim.x) s_wo[t] = __half2float(a.wout[t]);
    __syncthreads();
}

__global__ void __launch_bounds__(NL_THREADS) normals_train_fwd_kernel(const __grid_constant__ NlArgs a)
{
    __shared__ float s_w1[NL_HIDDEN * NL_IN], s_wo[NL_HIDDEN];
    nl_stage_weights(a, s_w1, s_wo);
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < nl_live(a)) nl_fwd_sample(a, s_w1, s_wo, i);
}

// Packed ray normal, warp = ray (composite_packed_fwd_kernel's layout): lanes over the ray's samples, a fixed shuffle tree.
__global__ void __launch_bounds__(256) normals_ray_sum_packed_kernel(const __grid_constant__ NlArgs a)
{
    const int lane = threadIdx.x & 31;
    const uint64_t ray = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (ray >= a.R) return;
    const int64_t b0 = a.offsets[ray], b1 = a.offsets[ray + 1];
    float s0 = 0.f, s1 = 0.f, s2 = 0.f;
    for (int64_t n = b0 + lane; n < b1; n += 32) {
        if (a.rinv[n] == 0.f) continue;
        const float w = a.w[n];
        s0 = fmaf(w, a.nrm[3 * n], s0); s1 = fmaf(w, a.nrm[3 * n + 1], s1); s2 = fmaf(w, a.nrm[3 * n + 2], s2);
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
        s0 += __shfl_xor_sync(0xffffffffu, s0, off); s1 += __shfl_xor_sync(0xffffffffu, s1, off); s2 += __shfl_xor_sync(0xffffffffu, s2, off);
    }
    if (lane == 0) { a.ray_nrm[3 * ray] = s0; a.ray_nrm[3 * ray + 1] = s1; a.ray_nrm[3 * ray + 2] = s2; }
}

__global__ void __launch_bounds__(128) normals_ray_sum_fixed_kernel(const __grid_constant__ NlArgs a)
{
    const uint64_t ray = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (ray < a.R) nl_ray_sum_fixed(a, ray);
}

// One CTA: pass 1 writes the unscaled dl/dN and reduces (sum l, #valid) in a fixed order, pass 2 scales by 1 / max(#valid, 1).
__global__ void __launch_bounds__(1024) normal_loss_kernel(const float* __restrict__ N, const float* __restrict__ gt, uint64_t R,
                                                           float* __restrict__ loss2, float* __restrict__ G)
{
    __shared__ float red[2][32];
    __shared__ float s_inv;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    float s_l = 0.f, s_c = 0.f;
    for (uint64_t r = tid; r < R; r += blockDim.x) {
        const float n3[3] = {N[3 * r], N[3 * r + 1], N[3 * r + 2]}, g3[3] = {gt[3 * r], gt[3 * r + 1], gt[3 * r + 2]};
        float l, dl[3];
        if (nl_loss_ray(n3, g3, l, dl)) { s_l += l; s_c += 1.f; }
        G[3 * r] = dl[0]; G[3 * r + 1] = dl[1]; G[3 * r + 2] = dl[2];
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) { s_l += __shfl_xor_sync(0xffffffffu, s_l, off); s_c += __shfl_xor_sync(0xffffffffu, s_c, off); }
    if (lane == 0) { red[0][warp] = s_l; red[1][warp] = s_c; }
    __syncthreads();
    if (warp == 0) {
        float l = lane < (int)(blockDim.x >> 5) ? red[0][lane] : 0.f, c = lane < (int)(blockDim.x >> 5) ? red[1][lane] : 0.f;
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) { l += __shfl_xor_sync(0xffffffffu, l, off); c += __shfl_xor_sync(0xffffffffu, c, off); }
        if (lane == 0) {
            const float inv = 1.f / fmaxf(c, 1.f);
            loss2[0] = l * inv; loss2[1] = c;
            s_inv = inv;
        }
    }
    __syncthreads();
    const float inv = s_inv;
    for (uint64_t r = tid; r < R; r += blockDim.x) { G[3 * r] *= inv; G[3 * r + 1] *= inv; G[3 * r + 2] *= inv; }
}

// Backward: grid-stride over tiles of NL_THREADS samples.  Each thread does one sample's table atomics and leaves its dg and mask
// in shared memory; then thread t adds the tile into its 8 entries of P (row t / 4, columns 8 (t % 4) ..) in registers.  P is
// flushed once per CTA.
__global__ void __launch_bounds__(NL_THREADS, 2) normals_train_bwd_kernel(const __grid_constant__ NlArgs a)
{
    __shared__ float s_w1[NL_HIDDEN * NL_IN], s_wo[NL_HIDDEN];
    __shared__ float s_dg[NL_THREADS][NL_IN + 1];
    __shared__ uint32_t s_m[NL_THREADS][2];
    nl_stage_weights(a, s_w1, s_wo);
    const int t = threadIdx.x, pj = t >> 2, pk0 = (t & 3) * 8;
    float P[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) P[q] = 0.f;
    const uint64_t live = nl_live(a);
    bool any_cta = false;
    for (uint64_t base = (uint64_t)blockIdx.x * NL_THREADS; base < live; base += (uint64_t)gridDim.x * NL_THREADS) {
        const uint64_t i = base + t;
        float dg[NL_IN]; uint32_t m[2] = {0u, 0u};
        const bool act = i < live && nl_bwd_sample(a, s_w1, s_wo, i, dg, m, nullptr);
        if (!__syncthreads_or(act)) continue;
        any_cta = true;
#pragma unroll
        for (int k = 0; k < NL_IN; ++k) s_dg[t][k] = act ? dg[k] : 0.f;
        s_m[t][0] = act ? m[0] : 0u; s_m[t][1] = act ? m[1] : 0u;
        __syncthreads();
#pragma unroll 4
        for (int s = 0; s < NL_THREADS; ++s) {
            const float mf = ((s_m[s][pj >> 5] >> (pj & 31)) & 1u) ? 1.f : 0.f;
#pragma unroll
            for (int q = 0; q < 8; ++q) P[q] = fmaf(mf, s_dg[s][pk0 + q], P[q]);
        }
        __syncthreads();
    }
    if (!any_cta) return;
    float dwo = nl_flush_row<8>(s_w1, s_wo, pj, pk0, P, a.dmlp);
    dwo += __shfl_xor_sync(0xffffffffu, dwo, 1);
    dwo += __shfl_xor_sync(0xffffffffu, dwo, 2);
    if ((t & 3) == 0 && dwo != 0.f) atomicAdd(a.dmlp + NL_HIDDEN * NL_IN + pj, dwo);
}

}  // namespace perf

using namespace perf;

static int setup_nl(const perf_grid_cfg* grid, const perf_mlp_cfg* mlp, const void* params_half, const perf_sample_layout* L,
                    const void* h1, const float* w, const float* T, float* nrm, float* rinv, NlArgs& a)
{
    PERF_CHECK_ARG(grid && mlp && params_half && L && h1 && w && T && nrm && rinv, "NULL pointer");
    memset(&a, 0, sizeof(a));
    uint64_t n_entries = 0;
    int rc = build_level_table(grid, &a.lt, &n_entries); if (rc) return rc;
    rc = check_mlp(mlp); if (rc) return rc;
    PERF_CHECK_SUP(a.lt.n_levels == NL_LEVELS && mlp->n_in == NL_IN && mlp->n_neurons == NL_HIDDEN && mlp->n_hidden_layers == 1 && mlp->n_out == 1,
                   "normal loss: the density network (16 levels, 32 -> 64 -> 1) only");
    uint64_t n_mlp = 0; rc = mlp_param_count(mlp, &n_mlp); if (rc) return rc;
    PERF_CHECK_ARG((uintptr_t)params_half % 16 == 0 && (uintptr_t)h1 % 16 == 0, "misaligned params / h1 (16 bytes)");
    const __half* ph = (const __half*)params_half;
    a.w1 = ph; a.wout = ph + NL_HIDDEN * NL_IN; a.table = (const __half2*)(ph + n_mlp);
    for (int d = 0; d < 3; ++d) { a.aabb_min[d] = L->aabb[d]; a.aabb_ext[d] = L->aabb[3 + d] - L->aabb[d]; }
    PERF_CHECK_ARG(a.aabb_ext[0] > 0.f && a.aabb_ext[1] > 0.f && a.aabb_ext[2] > 0.f, "empty aabb");
    a.R = L->R; a.N = L->N;
    a.h1 = (const __half*)h1; a.w = w; a.T = T; a.nrm = nrm; a.rinv = rinv;
    if (L->d_x01) {
        PERF_CHECK_ARG(L->d_offsets, "packed layout needs d_offsets");
        a.x01 = L->d_x01; a.offsets = L->d_offsets; a.ray_indices = L->d_ray_indices; a.n_dev = L->d_n_dev;
    } else {
        PERF_CHECK_ARG(L->d_rays_o && L->d_rays_d, "fixed-S layout needs d_rays_o / d_rays_d (or d_x01 for the packed layout)");
        PERF_CHECK_ARG(L->n_samples >= 1 && L->far > L->near && L->N == L->R * (uint64_t)L->n_samples, "fixed-S layout: N must be R * n_samples");
        PERF_CHECK_ARG(L->segments >= 1 && L->n_samples % L->segments == 0 && (L->segments == 1 || L->d_seg_trans), "bad segment count %u", L->segments);
        a.rays_o = L->d_rays_o; a.rays_d = L->d_rays_d; a.jitter = L->d_jitter; a.S = L->n_samples; a.seg = L->segments;
        a.near = L->near; a.far = L->far; a.seg_trans = L->d_seg_trans;
    }
    return PERF_OK;
}

extern "C" {
#pragma GCC visibility push(default)

int perf_normals_train_fwd(const perf_grid_cfg* grid, const perf_mlp_cfg* mlp, const void* d_params_half, const perf_sample_layout* layout,
                           const void* d_h1, const float* d_weights, const float* d_trans,
                           float* d_sample_normal, float* d_inv_norm, float* d_ray_normal, void* stream)
{
    NlArgs a;
    int rc = setup_nl(grid, mlp, d_params_half, layout, d_h1, d_weights, d_trans, d_sample_normal, d_inv_norm, a); if (rc) return rc;
    PERF_CHECK_ARG(d_ray_normal, "NULL pointer");
    a.ray_nrm = d_ray_normal;
    if (a.R == 0) return PERF_OK;
    if (a.N > 0) {
        normals_train_fwd_kernel<<<(unsigned)((a.N + NL_THREADS - 1) / NL_THREADS), NL_THREADS, 0, (cudaStream_t)stream>>>(a);
        PERF_LAUNCH_CHECK();
    }
    if (a.x01) normals_ray_sum_packed_kernel<<<(unsigned)((a.R * 32 + 255) / 256), 256, 0, (cudaStream_t)stream>>>(a);
    else normals_ray_sum_fixed_kernel<<<(unsigned)((a.R + 127) / 128), 128, 0, (cudaStream_t)stream>>>(a);
    PERF_LAUNCH_CHECK();
    return PERF_OK;
}

int perf_normal_loss(const float* d_ray_normal, const float* d_gt_normal, uint64_t R, float* d_loss2, float* d_g_ray_normal, void* stream)
{
    // a batch without rays has L_n = 0 and no valid ray; its [0,3] arrays may be NULL (an empty tensor's storage)
    PERF_CHECK_ARG(d_loss2 && (R == 0 || (d_ray_normal && d_gt_normal && d_g_ray_normal)), "NULL pointer");
    normal_loss_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(d_ray_normal, d_gt_normal, R, d_loss2, d_g_ray_normal);
    PERF_LAUNCH_CHECK();
    return PERF_OK;
}

int perf_normals_train_bwd(const perf_grid_cfg* grid, const perf_mlp_cfg* mlp, const void* d_params_half, const perf_sample_layout* layout,
                           const void* d_h1, const float* d_weights, const float* d_trans,
                           const float* d_sample_normal, const float* d_inv_norm, const float* d_g_ray_normal,
                           float* d_dparams, void* stream)
{
    NlArgs a;
    int rc = setup_nl(grid, mlp, d_params_half, layout, d_h1, d_weights, d_trans, const_cast<float*>(d_sample_normal),
                      const_cast<float*>(d_inv_norm), a); if (rc) return rc;
    PERF_CHECK_ARG(d_g_ray_normal && d_dparams, "NULL pointer");
    PERF_CHECK_ARG(!a.x01 || layout->d_ray_indices, "packed layout needs d_ray_indices");
    uint64_t n_mlp = 0; mlp_param_count(mlp, &n_mlp);
    PERF_CHECK_ARG((uintptr_t)(d_dparams + n_mlp) % 8 == 0, "misaligned grid gradient");
    a.g_ray = d_g_ray_normal; a.dmlp = d_dparams; a.dtable = (float2*)(d_dparams + n_mlp);
    if (a.R == 0 || a.N == 0) return PERF_OK;
    const uint64_t tiles = (a.N + NL_THREADS - 1) / NL_THREADS;
    const uint64_t cap = (uint64_t)num_sms() * 2;                 // two resident CTAs per SM (launch bounds)
    normals_train_bwd_kernel<<<(unsigned)(tiles < cap ? tiles : cap), NL_THREADS, 0, (cudaStream_t)stream>>>(a);
    PERF_LAUNCH_CHECK();
    return PERF_OK;
}

#ifdef PERF_HOST_HARNESS
/* TEST HARNESS ONLY (never compiled into libperfb200.so): the bodies above over HOST arrays, one thread, samples in order. */
static void host_weights(const NlArgs& a, float* w1, float* wo)
{
    for (int t = 0; t < NL_HIDDEN * NL_IN; ++t) w1[t] = __half2float(a.w1[t]);
    for (int t = 0; t < NL_HIDDEN; ++t) wo[t] = __half2float(a.wout[t]);
}

int perf_host_normals_train_fwd(const perf_grid_cfg* grid, const perf_mlp_cfg* mlp, const void* h_params_half, const perf_sample_layout* layout,
                                const void* h_h1, const float* h_weights, const float* h_trans,
                                float* h_sample_normal, float* h_inv_norm, float* h_ray_normal)
{
    NlArgs a;
    int rc = setup_nl(grid, mlp, h_params_half, layout, h_h1, h_weights, h_trans, h_sample_normal, h_inv_norm, a); if (rc) return rc;
    a.ray_nrm = h_ray_normal;
    static float w1[NL_HIDDEN * NL_IN], wo[NL_HIDDEN];
    host_weights(a, w1, wo);
    const uint64_t live = a.n_dev ? (uint64_t)*a.n_dev : a.N;
    for (uint64_t i = 0; i < live; ++i) nl_fwd_sample(a, w1, wo, i);
    for (uint64_t ray = 0; ray < a.R; ++ray) {
        if (!a.x01) { nl_ray_sum_fixed(a, ray); continue; }
        float s[3] = {0.f, 0.f, 0.f};
        for (int64_t n = a.offsets[ray]; n < a.offsets[ray + 1]; ++n)
            if (a.rinv[n] != 0.f) for (int d = 0; d < 3; ++d) s[d] = fmaf(a.w[n], a.nrm[3 * n + d], s[d]);
        for (int d = 0; d < 3; ++d) a.ray_nrm[3 * ray + d] = s[d];
    }
    return PERF_OK;
}

int perf_host_normal_loss(const float* h_ray_normal, const float* h_gt_normal, uint64_t R, float* h_loss2, float* h_g_ray_normal)
{
    float s_l = 0.f, s_c = 0.f;
    for (uint64_t r = 0; r < R; ++r) {
        const float n3[3] = {h_ray_normal[3 * r], h_ray_normal[3 * r + 1], h_ray_normal[3 * r + 2]};
        const float g3[3] = {h_gt_normal[3 * r], h_gt_normal[3 * r + 1], h_gt_normal[3 * r + 2]};
        float l, dl[3];
        if (nl_loss_ray(n3, g3, l, dl)) { s_l += l; s_c += 1.f; }
        for (int d = 0; d < 3; ++d) h_g_ray_normal[3 * r + d] = dl[d];
    }
    const float inv = 1.f / fmaxf(s_c, 1.f);
    h_loss2[0] = s_l * inv; h_loss2[1] = s_c;
    for (uint64_t k = 0; k < 3 * R; ++k) h_g_ray_normal[k] *= inv;
    return PERF_OK;
}

/* h_v [N,3] (dL/d grad01) and h_dg [N,32] (dL/dg) are optional per-sample outputs of the same bodies; h_dparams accumulates. */
int perf_host_normals_train_bwd(const perf_grid_cfg* grid, const perf_mlp_cfg* mlp, const void* h_params_half, const perf_sample_layout* layout,
                                const void* h_h1, const float* h_weights, const float* h_trans,
                                const float* h_sample_normal, const float* h_inv_norm, const float* h_g_ray_normal,
                                float* h_dparams, float* h_v, float* h_dg)
{
    NlArgs a;
    int rc = setup_nl(grid, mlp, h_params_half, layout, h_h1, h_weights, h_trans, const_cast<float*>(h_sample_normal),
                      const_cast<float*>(h_inv_norm), a); if (rc) return rc;
    uint64_t n_mlp = 0; mlp_param_count(mlp, &n_mlp);
    a.g_ray = h_g_ray_normal; a.dmlp = h_dparams; a.dtable = (float2*)(h_dparams + n_mlp);
    static float w1[NL_HIDDEN * NL_IN], wo[NL_HIDDEN];
    host_weights(a, w1, wo);
    static float P[NL_HIDDEN][NL_IN];
    memset(P, 0, sizeof(P));
    const uint64_t live = a.n_dev ? (uint64_t)*a.n_dev : a.N;
    for (uint64_t i = 0; i < live; ++i) {
        float dg[NL_IN]; uint32_t m[2];
        for (int k = 0; k < NL_IN; ++k) dg[k] = 0.f;
        const bool act = nl_bwd_sample(a, w1, wo, i, dg, m, h_v ? h_v + 3 * i : nullptr);
        if (h_dg) for (int k = 0; k < NL_IN; ++k) h_dg[NL_IN * i + k] = act ? dg[k] : 0.f;
        if (!act) continue;
        for (int j = 0; j < NL_HIDDEN; ++j)
            if ((m[j >> 5] >> (j & 31)) & 1u) for (int k = 0; k < NL_IN; ++k) P[j][k] += dg[k];
    }
    for (int j = 0; j < NL_HIDDEN; ++j) {
        const float dwo = nl_flush_row<NL_IN>(w1, wo, j, 0, P[j], h_dparams);
        h_dparams[NL_HIDDEN * NL_IN + j] += dwo;
    }
    return PERF_OK;
}
#endif

#pragma GCC visibility pop
}  // extern "C"
