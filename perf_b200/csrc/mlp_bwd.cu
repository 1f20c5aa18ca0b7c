// mlp_bwd.cu -- backward of the 64-wide bias-free MLP from the saved fp16 activations, ONE kernel on the
// Hopper tensor cores (wgmma; replaces tcnn FullyFusedMLP::backward_impl + its CUTLASS dW GEMMs for PeRF's two
// networks; the default path of ops.mlp_backward_half).  A CUDA-core twin (PERF_FLAG_SIMT_MLP) computes the same
// products from the same shared-memory operand images.
//
// Rows are samples (any order), thread t of a 128-thread CTA (one warpgroup) owns row t of the current 128-row tile.
//   colour net (two hidden layers), per tile:
//     dh2 = (dz Wout) . [h2 > 0]                    CUDA cores (n_out = 3)
//     D1  = dh2 W2          -> dh1 = D1 . [h1 > 0]  wgmma, A K-major, B = forward W2 image read MN-major; the mask is
//                                                   applied to the accumulator fragments, dh1 stored from them
//     D2  = dh1 W1          -> dfeat                wgmma, same; fragments -> fp32 row image -> row t
//     dW2 += dh2^T h1,  dW1 += dh1^T feat,  dWout^T += h2^T [dz|0]     wgmma, A and B MN-major
//   density net (one hidden layer): dh1 = (dz Wout) . [h1 > 0];  D2 = dh1 W1;  dW1 += dh1^T feat;  dWout^T += h1^T [dz|0]
// The weight-gradient accumulators stay in registers (wgmma fragments) for the whole kernel and are added to the
// global fp32 gradient once per CTA.  All operand images use the forward's no-swizzle K-major canonical layout
// (mlp_tc.cuh); "transposed" operands are the SAME images described as MN-major:
//     MN-major, no swizzle:  8 contiguous MN elements (16 B), 8 K-rows at 16 B stride, LBO = byte distance
//     between 8-row K groups (128), SBO = byte distance between 8-element MN groups (rows * 16)
// (canonical layout ((T,1,m),(8,k)):((1,T,SBO),(1T,LBO))), with the transpose immediates of wgmma selecting
// MN-major for A / B.
#include <stdlib.h>
#include "mlp_tc.cuh"

namespace perf {

struct MlpBwdArgs {
    const __half* w;         // flat fp16 MLP params (W1 [64,32] | W2 [64,64] (two hidden) | Wout [16,64])
    const uint4*  feat;      // [N,32] fp16
    const uint4*  h1;        // [N,64] fp16
    const uint4*  h2;        // [N,64] fp16 (two hidden) or NULL
    const float*  dz;        // [N,n_out] fp32: d loss / d output pre-activation
    uint64_t      N;
    float*        dW;        // flat fp32 gradient of the MLP params, accumulated (+=)
    float*        dfeat;     // [N,32] fp32
    uint32_t      n_out;     // 1..3
    uint32_t      dbg;       // bring-up only (flags >> 8): bit 0 swaps LBO / SBO of the MN-major descriptors (a negative control)
    const int64_t* n_dev;    // optional: the live row count in DEVICE memory (<= N = capacity); rows beyond it are skipped
};

// Fine-level grid scatter fused into the epilogue (perf_mlp_bwd_scatter): rows are the fixed-S training step's sample-major
// rows (row = k * R + ray); the thread that owns a row has its 32 feature gradients in registers and issues the reductions
// of levels [n_coarse, n_levels) itself, so that half of dfeat never goes to HBM and the L2-reduction-bound scatter overlaps
// the latency-bound MMA phases of the other resident CTAs.  The coarse levels keep their run-merging march kernel.
struct ScatterCtx {
    LevelTable lt;
    float aabb_min[3], aabb_ext[3];
    const float *rays_o, *rays_d, *jitter;
    uint64_t R; uint32_t S; float near, far;
    float2* dtable; uint32_t n_coarse;
};

// MN-major view of a canonical image with `rows` rows, K-step ks (16 rows)
__device__ __forceinline__ uint64_t desc_mn(uint32_t img, int rows, int ks, uint32_t dbg = 0)
{
    return (dbg & 1u) ? gmma_desc(img + ks * 256, (uint32_t)rows * 16u, 128u) : gmma_desc(img + ks * 256, 128u, (uint32_t)rows * 16u);
}
// K-major view of an activation image (128 rows), K-step ks (16 columns)
__device__ __forceinline__ uint64_t desc_k(uint32_t img, int ks) { return gmma_desc(img + ks * 2 * A_LBO, A_LBO, X_SBO); }

__host__ __device__ __forceinline__ float img_at(const uint8_t* img, int rows, int r, int c)
{
    return __half2float(*reinterpret_cast<const __half*>(img + ((c >> 3) * rows + r) * 16 + (c & 7) * 2));
}

// shared-memory map (bytes)
template <bool TWO> struct BwdSmem;
template <> struct BwdSmem<true> {
    static constexpr int DH2 = 0, DH1 = DH2 + A64_BYTES, H2 = DH1 + A64_BYTES, H1 = H2 + A64_BYTES, FEAT = H1 + A64_BYTES,
                         DZP = FEAT + A32_BYTES, W2 = DZP + 2 * TILE * 16, W1 = W2 + W64_BYTES, WOUT = W1 + W32_BYTES,
                         TOTAL = WOUT + 3 * HID * 4;
    static constexpr int N_G1 = 96, N_G2 = 16;
    static constexpr int GA = DH2 /* [DH2|DH1] */, GB = H1 /* [H1|FEAT] */;
};
template <> struct BwdSmem<false> {
    static constexpr int DH1 = 0, H1 = DH1 + A64_BYTES, FEAT = H1 + A64_BYTES, DZP = FEAT + A32_BYTES, W1 = DZP + 2 * TILE * 16,
                         WOUT = W1 + W32_BYTES, TOTAL = WOUT + 3 * HID * 4;
    static constexpr int N_G1 = 48;
    static constexpr int GA = DH1 /* [DH1|H1] */, GB = FEAT /* [FEAT|DZP] */;
    static constexpr int DH2 = 0, H2 = 0, W2 = 0, N_G2 = 0;      // unused with one hidden layer
};
constexpr int N_GACC = 112;       // CUDA-core twin of the weight-gradient accumulators: 96 (G1) + 16 (G2) columns of row t

template <int KGS>
__host__ __device__ __forceinline__ void store_row(uint8_t* img, int row, const uint4 (&v)[KGS])
{
#pragma unroll
    for (int kg = 0; kg < KGS; ++kg) *reinterpret_cast<uint4*>(img + (kg * TILE + row) * 16) = v[kg];
}
__host__ __device__ __forceinline__ uint32_t word_of(const uint4& q, int i) { return i == 0 ? q.x : i == 1 ? q.y : i == 2 ? q.z : q.w; }

// Output matrix as fp32 in the constant bank for the tensor-core kernel (same reason as c_wout in render.cu: the
// 64 * n_out multiplies per row then read their weight as c[bank][imm] instead of a broadcast shared-memory load;
// fewer shared-memory instructions in the MIO pipe).  Filled stream-ordered in front of every launch; one slot
// per device (launches for different networks on one device must not overlap in time).
__constant__ float c_wout_bwd[3 * HID];
__global__ void wout_bwd_to_const_kernel(const __half* __restrict__ wout, int n, float* __restrict__ dst)
{
    const int i = threadIdx.x;
    dst[i] = i < n ? __half2float(wout[i]) : 0.f;
}

// dh[j] = (h[j] > 0) ? sum_o dz[o] * wout[o][j] : 0, rounded to fp16, written as this thread's row of `dst`
template <bool CONSTW = false>
__host__ __device__ __forceinline__ void out_layer_backward(uint8_t* dst, int row, const uint4 (&h)[8], const float (&dz)[3], int n_out, const float* wout)
{
#pragma unroll
    for (int kg = 0; kg < 8; ++kg) {
        uint32_t o4[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const float2 hh = unpack_half2(word_of(h[kg], q));
            const int j = kg * 8 + 2 * q;
            float a = 0.f, b = 0.f;
#pragma unroll
            for (int o = 0; o < 3; ++o)
                if (o < n_out) {
#ifdef __CUDA_ARCH__
                    if constexpr (CONSTW) { a = fmaf(dz[o], c_wout_bwd[o * HID + j], a); b = fmaf(dz[o], c_wout_bwd[o * HID + j + 1], b); }
                    else
#endif
                    { a = fmaf(dz[o], wout[o * HID + j], a); b = fmaf(dz[o], wout[o * HID + j + 1], b); }
                }
            o4[q] = pack_half2(hh.x > 0.f ? a : 0.f, hh.y > 0.f ? b : 0.f);
        }
        *reinterpret_cast<uint4*>(dst + (kg * TILE + row) * 16) = make_uint4(o4[0], o4[1], o4[2], o4[3]);
    }
}

// ---- the per-thread phases of one tile (thread t = row t).  Between two phases every thread of the CTA must have
// finished the previous one (__syncthreads in the kernel, a loop over t in the host harness).

// phase 1: stage the saved activations and dz as operand images, output-layer backward on CUDA cores.
// Split in two so that the kernel can issue the global loads of tile i+1 (into registers) right after tile i has been
// staged: they are in flight during tile i's MMAs and epilogues instead of at the head of tile i+1.
template <bool TWO>
struct TileRegs { uint4 f4[4], h1v[8], hlast[TWO ? 8 : 1]; float dz[3]; };

template <bool TWO>
__host__ __device__ __forceinline__ void bwd_phase_load(const MlpBwdArgs& a, uint64_t tile, int t, TileRegs<TWO>& r)
{
    const uint64_t row = tile * TILE + t;
    const bool valid = row < a.N;
    const int n_out = (int)a.n_out;
    const uint4 z4 = make_uint4(0, 0, 0, 0);
#pragma unroll
    for (int q = 0; q < 4; ++q) r.f4[q] = valid ? a.feat[row * 4 + q] : z4;
#pragma unroll
    for (int q = 0; q < 8; ++q) r.h1v[q] = valid ? a.h1[row * 8 + q] : z4;
    if constexpr (TWO) {
#pragma unroll
        for (int q = 0; q < 8; ++q) r.hlast[q] = valid ? a.h2[row * 8 + q] : z4;
    }
#pragma unroll
    for (int o = 0; o < 3; ++o) r.dz[o] = (valid && o < n_out) ? a.dz[row * n_out + o] : 0.f;
}

template <bool TWO, bool CONSTW = false>
__host__ __device__ __forceinline__ void bwd_phase_store(uint8_t* smem, const float* s_wout, const MlpBwdArgs& a, int t, const TileRegs<TWO>& r)
{
    using L = BwdSmem<TWO>;
    const int n_out = (int)a.n_out;
    const uint4 z4 = make_uint4(0, 0, 0, 0);
    store_row(smem + L::FEAT, t, r.f4);
    store_row(smem + L::H1, t, r.h1v);
    // dz as 16 fp16 columns (cols >= n_out are zero)
    *reinterpret_cast<uint4*>(smem + L::DZP + (0 * TILE + t) * 16) = make_uint4(pack_half2(r.dz[0], r.dz[1]), pack_half2(r.dz[2], 0.f), 0u, 0u);
    *reinterpret_cast<uint4*>(smem + L::DZP + (1 * TILE + t) * 16) = z4;
    if constexpr (TWO) {
        uint4 hl[8];
#pragma unroll
        for (int q = 0; q < 8; ++q) hl[q] = r.hlast[q];
        store_row(smem + L::H2, t, hl);
        out_layer_backward<CONSTW>(smem + L::DH2, t, hl, r.dz, n_out, s_wout);
    } else {
        out_layer_backward<CONSTW>(smem + L::DH1, t, r.h1v, r.dz, n_out, s_wout);
    }
}

template <bool TWO>
__host__ __device__ __forceinline__ void bwd_phase_stage(uint8_t* smem, const float* s_wout, const MlpBwdArgs& a, uint64_t tile, int t)
{
    TileRegs<TWO> r;
    bwd_phase_load<TWO>(a, tile, t, r);
    bwd_phase_store<TWO>(smem, s_wout, a, t, r);
}

// CUDA-core twin of a data-gradient MMA: D[row][n0 + j] = sum_k A[row][k] * Wimg[k][n0 + j]
// (A: activation image, K-major; Wimg: forward weight image [64 rows k][n cols], i.e. the MN-major B operand)
__host__ __device__ __forceinline__ void simt_dgrad(const uint8_t* A, const uint8_t* Wimg, int row, int n0, float (&v)[32])
{
    for (int j = 0; j < 32; ++j) {
        float acc = 0.f;
        for (int k = 0; k < HID; ++k) acc = fmaf(img_at(A, TILE, row, k), img_at(Wimg, HID, k, n0 + j), acc);
        v[j] = acc;
    }
}

// phase 2 (two hidden layers): 32 columns [32c, 32c+32) of D1 = dh2 W2 -> dh1 = D1 . [h1 > 0] into the DH1 image
__host__ __device__ __forceinline__ void bwd_phase_hidden_chunk(uint8_t* smem, int t, int c, const float (&v)[32])
{
    using L = BwdSmem<true>;
    uint32_t p[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) {
        const uint4 hq = *reinterpret_cast<const uint4*>(smem + L::H1 + ((4 * c + j / 4) * TILE + t) * 16);
        const float2 hh = unpack_half2(word_of(hq, j % 4));
        p[j] = pack_half2(hh.x > 0.f ? v[2 * j] : 0.f, hh.y > 0.f ? v[2 * j + 1] : 0.f);
    }
#pragma unroll
    for (int q = 0; q < 4; ++q)
        *reinterpret_cast<uint4*>(smem + L::DH1 + ((4 * c + q) * TILE + t) * 16) = make_uint4(p[4 * q], p[4 * q + 1], p[4 * q + 2], p[4 * q + 3]);
}

// phase 3, CUDA-core twin of the weight-gradient MMAs: row m = t of G1 = [GA]^T [GB] (+= A[n][m] B[n][c] over the tile's
// rows) and G2; the tensor-core kernel computes only the blocks of G1 / G2 that bwd_flush_g1 / g2 use
template <bool TWO>
__host__ __device__ __forceinline__ void simt_wgrad(const uint8_t* smem, int t, float* gacc /* [N_GACC] of this thread */)
{
    using L = BwdSmem<TWO>;
    for (int c = 0; c < L::N_G1; ++c) {
        float acc = gacc[c];
        for (int n = 0; n < TILE; ++n) acc = fmaf(img_at(smem + L::GA, TILE, n, t), img_at(smem + L::GB, TILE, n, c), acc);
        gacc[c] = acc;
    }
    if constexpr (TWO) {
        for (int c = 0; c < L::N_G2; ++c) {
            float acc = gacc[96 + c];
            for (int n = 0; n < TILE; ++n) acc = fmaf(img_at(smem + L::H2, TILE, n, t), img_at(smem + L::DZP, TILE, n, c), acc);
            gacc[96 + c] = acc;
        }
    }
}

// phase 3: dfeat row from D2 = dh1 W1
__host__ __device__ __forceinline__ void bwd_phase_dfeat(const MlpBwdArgs& a, uint64_t tile, int t, const float (&v)[32])
{
    const uint64_t row = tile * TILE + t;
    if (row < a.N) {
        float4* dst = reinterpret_cast<float4*>(a.dfeat + row * 32);
#pragma unroll
        for (int q = 0; q < 8; ++q) dst[q] = make_float4(v[4 * q], v[4 * q + 1], v[4 * q + 2], v[4 * q + 3]);
    }
}

// reductions of the fine levels for one row; same position / weight / index arithmetic as bwd_rays_row_level (train.cu)
__device__ __forceinline__ void scatter_fine_levels(const ScatterCtx& c, uint64_t row, const float (&v)[32])
{
    const uint64_t ray = row % c.R; const uint32_t k = (uint32_t)(row / c.R);
    const float step = fixed_s_step(c.near, c.far, c.S);
    const float jit = c.jitter ? c.jitter[ray] : 0.f;
    const float ts = fixed_s_t(c.near, step, k, jit), te = fixed_s_t(c.near, step, k + 1, jit);
    const float tsum = __fadd_rn(ts, te);
    const float x = to_unit(sample_midpoint(c.rays_o[3 * ray], c.rays_d[3 * ray], tsum), c.aabb_min[0], c.aabb_ext[0]);
    const float y = to_unit(sample_midpoint(c.rays_o[3 * ray + 1], c.rays_d[3 * ray + 1], tsum), c.aabb_min[1], c.aabb_ext[1]);
    const float z = to_unit(sample_midpoint(c.rays_o[3 * ray + 2], c.rays_d[3 * ray + 2], tsum), c.aabb_min[2], c.aabb_ext[2]);
#pragma unroll
    for (int l = 8; l < 16; ++l) {                             // register indices of v must be compile-time: n_coarse == 8, 16 levels
        const float gx = v[2 * l], gy = v[2 * l + 1];
        if (gx == 0.f && gy == 0.f) continue;
        Corner8 cn;
        level_corners(c.lt, l, x, y, z, cn);
        float2 g8[8];
#pragma unroll
        for (int q = 0; q < 8; ++q) g8[q] = make_float2(cn.w[q] * gx, cn.w[q] * gy);
        scatter8<true>(c.dtable, cn.idx, g8);
    }
}

__host__ __device__ __forceinline__ void wgrad_add(float* p, float v)
{
#ifdef __CUDA_ARCH__
    atomicAdd(p, v);
#else
    *p += v;
#endif
}
// epilogue: 32 columns [c0, c0+32) of row m = t of G1 -> global gradient
template <bool TWO>
__host__ __device__ __forceinline__ void bwd_flush_g1(const MlpBwdArgs& a, int t, int c0, const float (&v)[32])
{
    using L = BwdSmem<TWO>;
    float* dW1 = a.dW;
    float* dW2 = a.dW + 64 * 32;
    float* dWo = a.dW + 64 * 32 + (TWO ? 64 * 64 : 0);
    for (int j = 0; j < 32; ++j) {
        const int c = c0 + j;
        if (c >= L::N_G1) break;
        if constexpr (TWO) {
            if (t < 64 && c < 64) wgrad_add(dW2 + t * 64 + c, v[j]);                               // dh2^T h1
            else if (t >= 64 && c >= 64) wgrad_add(dW1 + (t - 64) * 32 + (c - 64), v[j]);          // dh1^T feat
        } else {
            if (t < 64 && c < 32) wgrad_add(dW1 + t * 32 + c, v[j]);                               // dh1^T feat
            else if (t >= 64 && c >= 32 && c - 32 < (int)a.n_out) wgrad_add(dWo + (c - 32) * 64 + (t - 64), v[j]);   // h1^T dz
        }
    }
}
// epilogue (two hidden layers): row m = t of G2 = [h2|h1]^T [dz|0]
__host__ __device__ __forceinline__ void bwd_flush_g2(const MlpBwdArgs& a, int t, const float (&v)[32])
{
    float* dWo = a.dW + 64 * 32 + 64 * 64;
#pragma unroll
    for (int o = 0; o < 3; ++o) if (t < 64 && o < (int)a.n_out) wgrad_add(dWo + o * 64 + t, v[o]);
}

// Tensor-core kernel: the fp32 image of D2 (128 rows x 32 columns, 16 KB) over the DH1 image once the tile's MMAs are
// complete; float4 chunk q of row r at chunk (q ^ (r & 7)) so that row reads (8 threads, 8 rows) hit distinct banks
__device__ __forceinline__ float* d2_at(uint8_t* img, int r, int c)
{
    return reinterpret_cast<float*>(img) + r * 32 + ((((c >> 2) ^ (r & 7))) << 2) + (c & 3);
}

template <bool TWO, bool SIMT, bool FUSE = false>
__global__ void __launch_bounds__(128) mlp_bwd_kernel(const MlpBwdArgs a_in, const __grid_constant__ ScatterCtx sc)
{
    MlpBwdArgs a = a_in;
    if (a.n_dev) { const int64_t n = *a.n_dev; a.N = n < 0 ? 0 : ((uint64_t)n < a.N ? (uint64_t)n : a.N); }    // graph-replayable row count
    using L = BwdSmem<TWO>;
    extern __shared__ __align__(128) uint8_t smem[];
    float* s_wout = reinterpret_cast<float*>(smem + L::WOUT);
    const int t = threadIdx.x, warp = t >> 5, lane = t & 31;
    const uint32_t s0 = smem_u32(smem);

    // weights: forward canonical images (read MN-major by the dgrad MMAs) + fp32 output matrix
    load_weight_canonical(a.w, 32, smem + L::W1, t, TILE);
    const __half* wout_g = a.w + 64 * 32;
    if constexpr (TWO) { load_weight_canonical(a.w + 64 * 32, 64, smem + L::W2, t, TILE); wout_g += 64 * 64; }
    load_wout(wout_g, (int)a.n_out, s_wout, t, TILE);
    __syncthreads();
    float gacc[SIMT ? N_GACC : 1];
    if constexpr (SIMT) { for (int i = 0; i < N_GACC; ++i) gacc[i] = 0.f; }
    // tensor-core weight-gradient fragments (M = 64 rows of the gradient block): TWO: dW2 [64 x 64], dW1 [64 x 32],
    // dWout^T [64 x 8]; one hidden layer: dW1 [64 x 32], dWout^T [64 x 8]
    float g64[TWO ? 32 : 1], g32[16], g8[4];
#pragma unroll
    for (int i = 0; i < (TWO ? 32 : 1); ++i) g64[i] = 0.f;
#pragma unroll
    for (int i = 0; i < 16; ++i) g32[i] = 0.f;
#pragma unroll
    for (int i = 0; i < 4; ++i) g8[i] = 0.f;

    const uint64_t n_tiles = (a.N + TILE - 1) / TILE;
    bool first = true;
    TileRegs<TWO> regs;
    if (blockIdx.x < n_tiles) bwd_phase_load<TWO>(a, blockIdx.x, t, regs);
    for (uint64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x, first = false) {
        bwd_phase_store<TWO, !SIMT>(smem, s_wout, a, t, regs);          // tensor-core kernel: output matrix from the constant bank
        if (tile + gridDim.x < n_tiles) bwd_phase_load<TWO>(a, tile + gridDim.x, t, regs);     // in flight during this tile's MMAs
        if constexpr (!SIMT) fence_proxy_async();
        __syncthreads();

        if constexpr (TWO) {
            // ---- D1 = dh2 W2 -> dh1 = D1 . [h1 > 0]
            if constexpr (!SIMT) {
                // fragment (row, columns 8j + 2(lane%4) + {0,1}) -> the same position of DH1, masked by H1 there;
                // one M=64 half at a time (register budget of the accumulators)
#pragma unroll 1
                for (int h = 0; h < 2; ++h) {
                    float d[32];
#pragma unroll
                    for (int i = 0; i < 32; ++i) d[i] = 0.f;
                    wgmma_fence();
                    for (int ks = 0; ks < 4; ++ks)
                        wgmma_n64<0, 1>(d, desc_k(s0 + L::DH2 + h * 64 * 16, ks), desc_mn(s0 + L::W2, HID, ks, a.dbg), ks > 0 ? 1u : 0u);
                    wgmma_commit();
                    wgmma_wait();
#pragma unroll
                    for (int j = 0; j < 8; ++j)
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            const int off = j * A_LBO + (h * 64 + warp * 16 + (lane >> 2) + 8 * e) * 16 + (lane & 3) * 4;
                            const float2 hh = unpack_half2(*reinterpret_cast<const uint32_t*>(smem + L::H1 + off));
                            *reinterpret_cast<uint32_t*>(smem + L::DH1 + off) =
                                pack_half2(hh.x > 0.f ? d[4 * j + 2 * e] : 0.f, hh.y > 0.f ? d[4 * j + 2 * e + 1] : 0.f);
                        }
                }
                fence_proxy_async();
            } else {
#pragma unroll
                for (int c = 0; c < 2; ++c) {
                    float v[32];
                    simt_dgrad(smem + L::DH2, smem + L::W2, t, 32 * c, v);
                    bwd_phase_hidden_chunk(smem, t, c, v);
                }
            }
            __syncthreads();
        }

        // ---- D2 = dh1 W1 (-> dfeat) and the weight-gradient accumulations
        float v[32];
        if constexpr (!SIMT) {
            float d2[2][16];
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
                for (int i = 0; i < 16; ++i) d2[h][i] = 0.f;
            wgmma_fence();
#pragma unroll
            for (int h = 0; h < 2; ++h)
                for (int ks = 0; ks < 4; ++ks)
                    wgmma_n32<0, 1>(d2[h], desc_k(s0 + L::DH1 + h * 64 * 16, ks), desc_mn(s0 + L::W1, HID, ks, a.dbg), ks > 0 ? 1u : 0u);
            for (int ks = 0; ks < 8; ++ks) {
                if constexpr (TWO) {
                    wgmma_n64<1, 1>(g64, desc_mn(s0 + L::DH2, TILE, ks, a.dbg), desc_mn(s0 + L::H1, TILE, ks, a.dbg), 1u);
                    wgmma_n32<1, 1>(g32, desc_mn(s0 + L::DH1, TILE, ks, a.dbg), desc_mn(s0 + L::FEAT, TILE, ks, a.dbg), 1u);
                    wgmma_n8<1, 1>(g8, desc_mn(s0 + L::H2, TILE, ks, a.dbg), desc_mn(s0 + L::DZP, TILE, ks, a.dbg), 1u);
                } else {
                    wgmma_n32<1, 1>(g32, desc_mn(s0 + L::DH1, TILE, ks, a.dbg), desc_mn(s0 + L::FEAT, TILE, ks, a.dbg), 1u);
                    wgmma_n8<1, 1>(g8, desc_mn(s0 + L::H1, TILE, ks, a.dbg), desc_mn(s0 + L::DZP, TILE, ks, a.dbg), 1u);
                }
            }
            wgmma_commit();
            wgmma_wait();
            __syncthreads();                               // every MMA of the tile has read DH1
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
                for (int j = 0; j < 4; ++j)
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const int r = h * 64 + warp * 16 + (lane >> 2) + 8 * e, c = 8 * j + 2 * (lane & 3);
                        *reinterpret_cast<float2*>(d2_at(smem + L::DH1, r, c)) = make_float2(d2[h][4 * j + 2 * e], d2[h][4 * j + 2 * e + 1]);
                    }
            __syncthreads();
#pragma unroll
            for (int q = 0; q < 8; ++q) {
                const float4 f = *reinterpret_cast<const float4*>(d2_at(smem + L::DH1, t, 4 * q));
                v[4 * q] = f.x; v[4 * q + 1] = f.y; v[4 * q + 2] = f.z; v[4 * q + 3] = f.w;
            }
        } else {
            simt_wgrad<TWO>(smem, t, gacc);
            simt_dgrad(smem + L::DH1, smem + L::W1, t, 0, v);
        }
        if constexpr (FUSE) {
            const uint64_t row = tile * TILE + t;
            if (row < a.N) {
                // coarse half only, as LEVEL-MAJOR planes for the march kernel (plane l = float2 [N]): a warp of that
                // kernel reads one level of 32 neighbouring rays -- 256 contiguous bytes here, 32 sectors in [N, 32] rows
                float2* const planes = reinterpret_cast<float2*>(a.dfeat);
#pragma unroll
                for (int l = 0; l < 8; ++l) planes[(uint64_t)l * a.N + row] = make_float2(v[2 * l], v[2 * l + 1]);
                scatter_fine_levels(sc, row, v);
            }
        } else {
            bwd_phase_dfeat(a, tile, t, v);
        }
        __syncthreads();                                   // images are rewritten by the next tile
    }

    // ---- weight gradients of this CTA -> global
    if (!first) {
        if constexpr (SIMT) {
            for (int c0 = 0; c0 < L::N_G1; c0 += 32) {
                float v[32];
                for (int j = 0; j < 32; ++j) v[j] = (c0 + j < L::N_G1) ? gacc[c0 + j] : 0.f;
                bwd_flush_g1<TWO>(a, t, c0, v);
            }
            if constexpr (TWO) {
                float v[32];
                for (int j = 0; j < 32; ++j) v[j] = j < 16 ? gacc[96 + j] : 0.f;
                bwd_flush_g2(a, t, v);
            }
        } else {
            // fragment element i: row m = 16 warp + lane/4 + 8 ((i/2) & 1), column n = 8 (i/4) + 2 (lane%4) + (i & 1)
            float* dW1 = a.dW;
            float* dWo = a.dW + 64 * 32 + (TWO ? 64 * 64 : 0);
            const int m0 = warp * 16 + (lane >> 2), n0 = 2 * (lane & 3);
            if constexpr (TWO) {
                float* dW2 = a.dW + 64 * 32;
#pragma unroll
                for (int i = 0; i < 32; ++i) atomicAdd(dW2 + (m0 + 8 * ((i >> 1) & 1)) * 64 + 8 * (i >> 2) + n0 + (i & 1), g64[i]);
            }
#pragma unroll
            for (int i = 0; i < 16; ++i) atomicAdd(dW1 + (m0 + 8 * ((i >> 1) & 1)) * 32 + 8 * (i >> 2) + n0 + (i & 1), g32[i]);
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int o = n0 + (i & 1);
                if (o < (int)a.n_out) atomicAdd(dWo + o * 64 + m0 + 8 * ((i >> 1) & 1), g8[i]);
            }
        }
    }
}

template <bool TWO, bool SIMT, bool FUSE = false>
static int launch_mlp_bwd(const MlpBwdArgs& a, cudaStream_t stream, const ScatterCtx* scp = nullptr)
{
    auto k = mlp_bwd_kernel<TWO, SIMT, FUSE>;
    static ScatterCtx sc_none;                                  // zero-initialised: unused when !FUSE
    const ScatterCtx& sc = scp ? *scp : sc_none;
    static thread_local int attr_dev = -1, per_sm = 1;
    int dev = 0; PERF_CUDA(cudaGetDevice(&dev));
    if (attr_dev != dev) {
        PERF_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, BwdSmem<TWO>::TOTAL));
        // resident CTAs per SM: registers (the weight-gradient fragments) and shared memory decide -- queried, not assumed
        PERF_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k, TILE, BwdSmem<TWO>::TOTAL));
        if (per_sm < 1) per_sm = 1;
        attr_dev = dev;
    }
    if (!SIMT) {
        static thread_local int sym_dev = -1; static thread_local float* sym = nullptr;
        if (sym_dev != dev) { PERF_CUDA(cudaGetSymbolAddress((void**)&sym, c_wout_bwd)); sym_dev = dev; }
        wout_bwd_to_const_kernel<<<1, 3 * HID, 0, stream>>>(a.w + 64 * 32 + (TWO ? 64 * 64 : 0), (int)a.n_out * HID, sym);
        PERF_LAUNCH_CHECK();
    }
    const uint64_t n_tiles = (a.N + TILE - 1) / TILE;
    const uint64_t slots = (uint64_t)num_sms() * (uint64_t)per_sm;              // one wave of persistent CTAs
    k<<<(unsigned)(n_tiles < slots ? n_tiles : slots), TILE, BwdSmem<TWO>::TOTAL, stream>>>(a, sc);
    PERF_LAUNCH_CHECK();
    return PERF_OK;
}

}  // namespace perf

using namespace perf;

#ifdef PERF_HOST_HARNESS
/* TEST HARNESS ONLY (never compiled into libperfb200.so): one CTA of the CUDA-core twin emulated on the host -- the
 * per-thread phases above run for t = 0..127 where the kernel has a __syncthreads -- over HOST arrays.  It checks
 * the operand images, the transposed reads, the block layout of the weight-gradient accumulators and the flush;
 * only the wgmma descriptors themselves need a GPU. */
template <bool TWO>
static void host_mlp_bwd(const MlpBwdArgs& a, uint8_t* smem, float* gacc /* [128][N_GACC] */)
{
    using L = BwdSmem<TWO>;
    float* s_wout = reinterpret_cast<float*>(smem + L::WOUT);
    auto load_w = [&](const __half* gW, int K, uint8_t* dst) {      // load_weight_canonical
        for (int c = 0; c < HID * (K / 8); ++c) { const int n = c % HID, kg = c / HID;
            *reinterpret_cast<uint4*>(dst + (kg * HID + n) * 16) = *reinterpret_cast<const uint4*>(gW + (size_t)n * K + kg * 8); }
    };
    load_w(a.w, 32, smem + L::W1);
    const __half* wout_g = a.w + 64 * 32;
    if (TWO) { load_w(a.w + 64 * 32, 64, smem + L::W2); wout_g += 64 * 64; }
    for (int c = 0; c < (int)a.n_out * HID; ++c) s_wout[c] = __half2float(wout_g[c]);
    const uint64_t n_tiles = (a.N + TILE - 1) / TILE;
    for (uint64_t tile = 0; tile < n_tiles; ++tile) {
        for (int t = 0; t < TILE; ++t) bwd_phase_stage<TWO>(smem, s_wout, a, tile, t);
        if (TWO) {
            float v[TILE][2][32];
            for (int t = 0; t < TILE; ++t) for (int c = 0; c < 2; ++c) simt_dgrad(smem + L::DH2, smem + L::W2, t, 32 * c, v[t][c]);
            for (int t = 0; t < TILE; ++t) for (int c = 0; c < 2; ++c) bwd_phase_hidden_chunk(smem, t, c, v[t][c]);
        }
        for (int t = 0; t < TILE; ++t) {
            simt_wgrad<TWO>(smem, t, gacc + t * N_GACC);
            float v[32];
            simt_dgrad(smem + L::DH1, smem + L::W1, t, 0, v);
            bwd_phase_dfeat(a, tile, t, v);
        }
    }
    for (int t = 0; t < TILE; ++t) {
        for (int c0 = 0; c0 < L::N_G1; c0 += 32) {
            float v[32];
            for (int j = 0; j < 32; ++j) v[j] = (c0 + j < L::N_G1) ? gacc[t * N_GACC + c0 + j] : 0.f;
            bwd_flush_g1<TWO>(a, t, c0, v);
        }
        if (TWO) {
            float v[32];
            for (int j = 0; j < 32; ++j) v[j] = j < 16 ? gacc[t * N_GACC + 96 + j] : 0.f;
            bwd_flush_g2(a, t, v);
        }
    }
}

#endif

extern "C" {
#pragma GCC visibility push(default)

int perf_mlp_bwd(const perf_mlp_cfg* mlp, const void* d_weights_half, const void* d_feat, const void* d_h1, const void* d_h2,
                 const float* d_dz, uint64_t N, const int64_t* d_n_dev, float* d_dweights, float* d_dfeat, uint32_t flags, void* stream)
{
    int rc = check_mlp(mlp); if (rc) return rc;
    PERF_CHECK_ARG(d_weights_half && d_feat && d_h1 && d_dz && d_dweights && d_dfeat, "NULL pointer");
    PERF_CHECK_ARG(mlp->n_hidden_layers == 1 || d_h2, "two hidden layers need d_h2");
    PERF_CHECK_SUP(mlp->n_out <= 3, "n_out=%u (the backward kernel implements 1..3 outputs)", mlp->n_out);
    PERF_CHECK_ARG(((uintptr_t)d_weights_half | (uintptr_t)d_feat | (uintptr_t)d_h1 | (uintptr_t)d_h2 | (uintptr_t)d_dfeat) % 16 == 0, "misaligned buffer");
    if (N == 0) return PERF_OK;
    MlpBwdArgs a;
    a.w = (const __half*)d_weights_half; a.feat = (const uint4*)d_feat; a.h1 = (const uint4*)d_h1; a.h2 = (const uint4*)d_h2;
    a.dz = d_dz; a.N = N; a.dW = d_dweights; a.dfeat = d_dfeat; a.n_out = mlp->n_out; a.dbg = flags >> 8; a.n_dev = d_n_dev;
    const bool simt = (flags & PERF_FLAG_SIMT_MLP) != 0;
    if (mlp->n_hidden_layers == 2) return simt ? launch_mlp_bwd<true, true>(a, (cudaStream_t)stream) : launch_mlp_bwd<true, false>(a, (cudaStream_t)stream);
    return simt ? launch_mlp_bwd<false, true>(a, (cudaStream_t)stream) : launch_mlp_bwd<false, false>(a, (cudaStream_t)stream);
}

int perf_mlp_bwd_scatter(const perf_mlp_cfg* mlp, const void* d_weights_half, const void* d_feat, const void* d_h1, const void* d_h2,
                         const float* d_dz, uint64_t N, float* d_dweights, float* d_dfeat,
                         const perf_grid_cfg* grid, const float* aabb6, const float* d_rays_o, const float* d_rays_d, const float* d_jitter,
                         uint64_t R, uint32_t n_samples, float near, float far, float* d_dtable, void* stream)
{
    int rc = check_mlp(mlp); if (rc) return rc;
    PERF_CHECK_ARG(d_weights_half && d_feat && d_h1 && d_dz && d_dweights && d_dfeat && grid && aabb6 && d_rays_o && d_rays_d && d_dtable, "NULL pointer");
    PERF_CHECK_ARG(mlp->n_hidden_layers == 1 || d_h2, "two hidden layers need d_h2");
    PERF_CHECK_SUP(mlp->n_out <= 3, "n_out=%u (the backward kernel implements 1..3 outputs)", mlp->n_out);
    PERF_CHECK_ARG(((uintptr_t)d_weights_half | (uintptr_t)d_feat | (uintptr_t)d_h1 | (uintptr_t)d_h2 | (uintptr_t)d_dfeat | (uintptr_t)d_dtable) % 16 == 0, "misaligned buffer");
    PERF_CHECK_ARG(N == R * (uint64_t)n_samples && n_samples >= 1 && far > near, "rows must be the R x S sample-major rows of a fixed-S step");
    if (N == 0) return PERF_OK;
    ScatterCtx sc; memset(&sc, 0, sizeof(sc));
    rc = build_level_table(grid, &sc.lt, nullptr); if (rc) return rc;
    PERF_CHECK_SUP(sc.lt.n_levels == 16, "fused scatter needs n_levels == 16 (got %u)", sc.lt.n_levels);
    for (int i = 0; i < 3; ++i) { sc.aabb_min[i] = aabb6[i]; sc.aabb_ext[i] = aabb6[3 + i] - aabb6[i]; }
    sc.rays_o = d_rays_o; sc.rays_d = d_rays_d; sc.jitter = d_jitter; sc.R = R; sc.S = n_samples; sc.near = near; sc.far = far;
    sc.dtable = (float2*)d_dtable; sc.n_coarse = 8;
    MlpBwdArgs a;
    a.w = (const __half*)d_weights_half; a.feat = (const uint4*)d_feat; a.h1 = (const uint4*)d_h1; a.h2 = (const uint4*)d_h2;
    a.dz = d_dz; a.N = N; a.dW = d_dweights; a.dfeat = d_dfeat; a.n_out = mlp->n_out; a.dbg = 0; a.n_dev = nullptr;
    if (mlp->n_hidden_layers == 2) return launch_mlp_bwd<true, false, true>(a, (cudaStream_t)stream, &sc);
    return launch_mlp_bwd<false, false, true>(a, (cudaStream_t)stream, &sc);
}

#ifdef PERF_HOST_HARNESS
/* TEST HARNESS ONLY: see host_mlp_bwd above. */
int perf_host_mlp_bwd(const perf_mlp_cfg* mlp, const void* h_weights_half, const void* h_feat, const void* h_h1, const void* h_h2,
                      const float* h_dz, uint64_t N, float* h_dweights, float* h_dfeat)
{
    int rc = check_mlp(mlp); if (rc) return rc;
    PERF_CHECK_ARG(h_weights_half && h_feat && h_h1 && h_dz && h_dweights && h_dfeat && (mlp->n_hidden_layers == 1 || h_h2), "NULL pointer");
    PERF_CHECK_SUP(mlp->n_out <= 3, "n_out=%u", mlp->n_out);
    MlpBwdArgs a;
    a.w = (const __half*)h_weights_half; a.feat = (const uint4*)h_feat; a.h1 = (const uint4*)h_h1; a.h2 = (const uint4*)h_h2;
    a.dz = h_dz; a.N = N; a.dW = h_dweights; a.dfeat = h_dfeat; a.n_out = mlp->n_out; a.dbg = 0; a.n_dev = nullptr;
    uint8_t* smem = (uint8_t*)aligned_alloc(128, (size_t)(BwdSmem<true>::TOTAL + 127) / 128 * 128);
    float* gacc = (float*)calloc((size_t)TILE * N_GACC, sizeof(float));
    if (!smem || !gacc) { free(smem); free(gacc); return PERF_ECUDA; }
    if (mlp->n_hidden_layers == 2) host_mlp_bwd<true>(a, smem, gacc); else host_mlp_bwd<false>(a, smem, gacc);
    free(smem); free(gacc);
    return PERF_OK;
}
#endif

#pragma GCC visibility pop
}  // extern "C"
