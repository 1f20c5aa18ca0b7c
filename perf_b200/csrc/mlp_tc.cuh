// mlp_tc.cuh -- building blocks of the 64-wide bias-free MLP on the Hopper tensor cores (wgmma).
//
// One warpgroup = 128 threads = one 128-row tile; thread t owns row t: it produces the row's fp16 input
// features and runs the row's epilogue.  A layer is two M=64 wgmma chains (rows 0-63, 64-127) whose fp32 accumulator
// fragments are rounded (ReLU, fp16) in registers and written straight into the next layer's operand image, from
// which every thread then reads its own row back (layer_relu).  The eval renders skip that round trip after layer 1: the
// rounded fragments ARE the next layer's A operand in registers (relu_frag, render.cu::eval_mlp_regs).
//
// Operand layout in shared memory (both A = activations and B = weights): K-major, NO swizzle,
// i.e. the canonical "interleaved" layout of 8x16-byte core matrices:
//     element (row r, col k)  ->  byte  (k/8) * LBO + r * 16 + (k%8) * 2
// with LBO = rows*16 (all rows of one 8-column k-group are contiguous) and SBO = 128 (8 rows).
// A thread therefore writes its row as K/8 16-byte chunks at stride LBO: consecutive threads
// hit consecutive 16-byte slots -> conflict-free STS.128, no swizzle arithmetic.  The fragment stores of a
// layer (one column pair of 8 rows x 4 pairs per warp and instruction) cover 128 contiguous bytes: conflict-free too.
#pragma once
#include "common.cuh"

namespace perf {

constexpr int      TILE  = 128;          // rows per tile (two wgmma M=64 halves)
constexpr int      HID   = 64;           // hidden width (wgmma N)
constexpr uint32_t A_LBO = TILE * 16;    // 2048 B between k-groups of an activation tile
constexpr uint32_t W_LBO = HID * 16;     // 1024 B between k-groups of a weight matrix
constexpr uint32_t X_SBO = 128;          // 8 rows * 16 B

constexpr int A32_BYTES = 4 * TILE * 16; //  8 KB : 128 x 32 fp16
constexpr int A64_BYTES = 8 * TILE * 16; // 16 KB : 128 x 64 fp16
constexpr int W32_BYTES = 4 * HID * 16;  //  4 KB :  64 x 32 fp16
constexpr int W64_BYTES = 8 * HID * 16;  //  8 KB :  64 x 64 fp16

// Barrier of this thread's warpgroup only (named barrier 1 + threadIdx.x / 128, 128 threads): the field kernels run up to
// four independent 128-row tiles per CTA, one per warpgroup, and a tile's barriers must not wait for the others.  In a
// 128-thread CTA it is equivalent to __syncthreads().
__device__ __forceinline__ void wg_sync()
{
    asm volatile("bar.sync %0, 128;" :: "r"(1 + (int)(threadIdx.x >> 7)) : "memory");
}

// [64, K] row-major fp16 weights in global memory -> canonical K-major smem layout.
__device__ __forceinline__ void load_weight_canonical(const __half* __restrict__ gW, int K, uint8_t* dst, int tid, int nthreads)
{
    const int kgs = K / 8;
    for (int c = tid; c < HID * kgs; c += nthreads) {
        const int n = c % HID, kg = c / HID;
        const uint4 v = *reinterpret_cast<const uint4*>(gW + (size_t)n * K + kg * 8);
        *reinterpret_cast<uint4*>(dst + (kg * HID + n) * 16) = v;
    }
}
// last matrix [16 (padded), 64] fp16 -> fp32 [n_out][64] (fp16 -> fp32 is exact)
__device__ __forceinline__ void load_wout(const __half* __restrict__ gW, int n_out, float* dst, int tid, int nthreads)
{
    for (int c = tid; c < n_out * HID; c += nthreads) dst[c] = __half2float(gW[c]);
}

__device__ __forceinline__ float dot8(uint4 a, uint4 w, float acc)
{
    const uint32_t av[4] = {a.x, a.y, a.z, a.w}, wv[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        const float2 fa = unpack_half2(av[q]), fw = unpack_half2(wv[q]);
        acc = fmaf(fa.x, fw.x, acc); acc = fmaf(fa.y, fw.y, acc);
    }
    return acc;
}

// 32 accumulator columns [32c, 32c+32) of this thread's row on CUDA cores (debug path, PERF_FLAG_SIMT_MLP): computed
// from the very same shared-memory operands the tensor cores read, so a layout bug shows up as a TC-vs-SIMT mismatch.
__device__ __forceinline__ void simt_chunk(int c, int K, const uint8_t* A, const uint8_t* W, int row, float (&v)[32])
{
#pragma unroll 1
    for (int j = 0; j < 32; ++j) {
        const int n = 32 * c + j;
        float acc = 0.f;
        for (int kg = 0; kg < K / 8; ++kg)
            acc = dot8(*reinterpret_cast<const uint4*>(A + (kg * TILE + row) * 16),
                       *reinterpret_cast<const uint4*>(W + (kg * HID + n) * 16), acc);
        v[j] = acc;
    }
}

// ReLU + round to fp16 (tcnn keeps hidden activations in __half), two values per instruction:
// cvt.rn.relu.f16x2.f32 rounds a pair and clamps it at zero in ONE instruction (round(max(x,0)) == max(round(x),0);
// until round 2 this was F2FP + HMNMX2, 96 more instructions per sample in the render kernel).
__device__ __forceinline__ void relu_pack(const float (&v)[32], uint32_t (&p)[16])
{
#pragma unroll
    for (int j = 0; j < 16; ++j)
        asm("cvt.rn.relu.f16x2.f32 %0, %1, %2;" : "=r"(p[j]) : "f"(v[2 * j + 1]), "f"(v[2 * j]));     // d = {hi: a, lo: b}
}

__device__ __forceinline__ uint32_t relu_pack2(float lo, float hi)
{
    uint32_t p; asm("cvt.rn.relu.f16x2.f32 %0, %1, %2;" : "=r"(p) : "f"(hi), "f"(lo)); return p;
}

// m64n64 fp32 accumulator fragment -> ReLU-rounded fp16 A fragments of the next layer, without leaving the registers:
// register j of k-slice s (a[4s + j], columns [16s, 16s + 16)) is the accumulator pair (8s + 2j, 8s + 2j + 1).
__device__ __forceinline__ void relu_frag(const float (&d)[32], uint32_t (&a)[16])
{
#pragma unroll
    for (int i = 0; i < 16; ++i) a[i] = relu_pack2(d[2 * i], d[2 * i + 1]);
}

// acc.x += a.x * b.x, acc.y += a.y * b.y: two independent fp32 FMAs (the even / odd partial sums of out_dots)
__device__ __forceinline__ void fma2(float2& acc, float2 a, float2 b)
{
    acc.x = fmaf(a.x, b.x, acc.x); acc.y = fmaf(a.y, b.y, acc.y);
}

// write 32 packed fp16 values as k-groups [kg0, kg0+4) of this thread's row of an activation tile
__device__ __forceinline__ void store_chunk_canonical(uint8_t* A, int row, int kg0, const uint32_t (&p)[16])
{
#pragma unroll
    for (int q = 0; q < 4; ++q)
        *reinterpret_cast<uint4*>(A + ((kg0 + q) * TILE + row) * 16) = make_uint4(p[4 * q], p[4 * q + 1], p[4 * q + 2], p[4 * q + 3]);
}
// same 32 values to a row-major [N,64] fp16 global buffer (activation save for the backward pass)
__device__ __forceinline__ void store_chunk_global(uint4* row_ptr /* 8 uint4 per row */, int c, const uint32_t (&p)[16])
{
#pragma unroll
    for (int q = 0; q < 4; ++q)
        row_ptr[4 * c + q] = make_uint4(p[4 * q], p[4 * q + 1], p[4 * q + 2], p[4 * q + 3]);
}

// this thread's row, columns [32c, 32c+32), of a canonical 128 x 64 fp16 image as 16 packed pairs
__device__ __forceinline__ void load_chunk_canonical(const uint8_t* A, int row, int c, uint32_t (&p)[16])
{
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        const uint4 u = *reinterpret_cast<const uint4*>(A + ((4 * c + q) * TILE + row) * 16);
        p[4 * q] = u.x; p[4 * q + 1] = u.y; p[4 * q + 2] = u.z; p[4 * q + 3] = u.w;
    }
}

// One hidden layer, all 128 threads: dst (canonical 128 x 64 fp16 image) = fp16(ReLU(A[128 x K] W[64 x K]^T)).
// Before: A and W are written and made visible to the async proxy (fence_proxy_async + barrier).  After: a barrier
// before any thread reads another thread's rows of dst.  OVERLAP: dst overlaps A (a barrier separates the last
// read of A from the first store).
template <bool SIMT, bool OVERLAP = false>
__device__ __forceinline__ void layer_relu(uint8_t* dst, const uint8_t* A, const uint8_t* W, int K, int tid)
{
    if constexpr (SIMT) {
        uint32_t hp[2][16];
#pragma unroll
        for (int c = 0; c < 2; ++c) {
            float v[32];
            simt_chunk(c, K, A, W, tid, v);
            relu_pack(v, hp[c]);
        }
        if constexpr (OVERLAP) wg_sync();
#pragma unroll
        for (int c = 0; c < 2; ++c) store_chunk_canonical(dst, tid, 4 * c, hp[c]);
    } else {
        const int warp = tid >> 5, lane = tid & 31;
        float d[2][32];
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int i = 0; i < 32; ++i) d[h][i] = 0.f;
        wgmma_fence();
#pragma unroll
        for (int h = 0; h < 2; ++h)
            for (int ks = 0; ks < K / 16; ++ks)
                wgmma_n64<0, 0>(d[h], gmma_desc(smem_u32(A) + h * 64 * 16 + ks * 2 * A_LBO, A_LBO, X_SBO),
                                gmma_desc(smem_u32(W) + ks * 2 * W_LBO, W_LBO, X_SBO), ks > 0 ? 1u : 0u);
        wgmma_commit();
        wgmma_wait();
        if constexpr (OVERLAP) wg_sync();
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            uint8_t* const p = dst + (h * 64 + warp * 16 + (lane >> 2)) * 16 + (lane & 3) * 4;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                *reinterpret_cast<uint32_t*>(p + j * A_LBO) = relu_pack2(d[h][4 * j], d[h][4 * j + 1]);
                *reinterpret_cast<uint32_t*>(p + j * A_LBO + 8 * 16) = relu_pack2(d[h][4 * j + 2], d[h][4 * j + 3]);
            }
        }
    }
}

// Output layer on CUDA cores (n_out is 1 or 3: a padded N=16 MMA + another smem round trip would cost more than the
// 64*n_out FMAs per row).  Every output keeps TWO partial sums -- acc[o].x over the even hidden units, acc[o].y over
// the odd ones, in increasing order -- one pair per packed pair of activations; the pre-activation is
// acc[o].x + acc[o].y (out_sum).  network_fwd_kernel, the training forward (render.cu, SAVE = 1/2), the SIMT twin and the
// legacy scan kernel share this order; the eval renders (render.cu::eval_mlp_regs) sum the output layers on the tensor cores.
//   acc[o] += h[32c + 2j, 32c + 2j + 1] * wout[o][32c + 2j, 32c + 2j + 1]      (wout: fp32 in shared memory)
template <int NOUT_MAX>
__device__ __forceinline__ void out_dots(const uint32_t (&p)[16], const float* wout, int c, int n_out, float2 (&acc)[NOUT_MAX])
{
    float2 v[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) v[j] = unpack_half2(p[j]);
#pragma unroll
    for (int o = 0; o < NOUT_MAX; ++o) {
        if (o < n_out) {
            const float4* w4 = reinterpret_cast<const float4*>(wout + o * HID + 32 * c);
            float2 a = acc[o];
#pragma unroll
            for (int q = 0; q < 8; ++q) {
                const float4 w = w4[q];
                fma2(a, v[2 * q], make_float2(w.x, w.y));
                fma2(a, v[2 * q + 1], make_float2(w.z, w.w));
            }
            acc[o] = a;
        }
    }
}
__device__ __forceinline__ float out_sum(float2 acc) { return __fadd_rn(acc.x, acc.y); }

// tcnn output: pre-activation rounded to fp16, activation in fp32, result rounded to fp16
__device__ __forceinline__ float finish_output(float acc, uint32_t out_act)
{
    float o = round_half(acc);
    if (out_act == 1) o = round_half(1.0f / (1.0f + expf(-o)));
    return o;
}

}  // namespace perf
