// grid_grad.cuh -- per-level derivative of the hash-grid encode w.r.t. the input position, shared by the input-gradient
// kernels (encoding_grad.cu) and the surface-normal pass of the eval renderers (render.cu).
//
// Per level, with p = fract(scale*x + 0.5), s = p (Linear) or p^2(3-2p) (Smoothstep), omega_1 = s,
// omega_0 = 1-s and v_c the table entry of corner c:
//     y      = sum_c  prod_d omega_{c_d}(s_d) * v_c
//     dy/dx_d          = scale   * s'(p_d)          * A_d ,  A_d  = sum_{other two dims} omega*omega * (v_right - v_left)
//     d2y/dx_d^2       = scale^2 * s''(p_d)         * A_d
//     d2y/dx_d dx_e    = scale^2 * s'(p_d) s'(p_e)  * B_de,  B_de = sum_{third dim} omega * (v_11 - v_10 - v_01 + v_00)
// Everything is __host__ __device__ so that tests/host_harness.py runs the same bodies on the CPU.
#pragma once
#include "common.cuh"

namespace perf {

struct LevelFrame {
    uint32_t idx[8];          // absolute entry index of corner c (bit0=x, bit1=y, bit2=z)
    float s[3], ds[3], dds[3];
    float scale;
};

__host__ __device__ __forceinline__ void level_frame(const LevelTable& lt, int l, float x, float y, float z, LevelFrame& f)
{
    const float scale = lt.scale[l];
    const uint32_t res = lt.res[l], size = lt.size[l], off = lt.offset[l];
    const bool hashed = (lt.hashed_mask >> l) & 1u, pow2 = (lt.pow2_mask >> l) & 1u;
    const float in[3] = {x, y, z};
    uint32_t g[3];
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        // common.cuh::cell_frame per axis, kept inline: calling it changes the register allocation of encoding_grad.cu
        const float pos = fmaf(scale, in[d], 0.5f), fl = floorf(pos), p = pos - fl;
        g[d] = (uint32_t)(int)fl;
        if (lt.smoothstep) { f.s[d] = p * p * (3.0f - 2.0f * p); f.ds[d] = 6.0f * p * (1.0f - p); f.dds[d] = 6.0f - 12.0f * p; }
        else               { f.s[d] = p;                         f.ds[d] = 1.0f;                 f.dds[d] = 0.0f; }
    }
#pragma unroll
    for (int k = 0; k < 8; ++k)
        f.idx[k] = off + level_index(g[0] + (k & 1), g[1] + ((k >> 1) & 1), g[2] + ((k >> 2) & 1), hashed, pow2, res, size);
    f.scale = scale;
}

// A_d of both features: sum over the corners of the other two dims of omega*omega*(v_right - v_left)
template <int D>
__host__ __device__ __forceinline__ float2 diff_along(const LevelFrame& f, const float2 (&v)[8])
{
    constexpr int E = (D + 1) % 3, H = (D + 2) % 3;
    float2 a = make_float2(0.f, 0.f);
#pragma unroll
    for (int ce = 0; ce < 2; ++ce)
#pragma unroll
        for (int ch = 0; ch < 2; ++ch) {
            const float w = (ce ? f.s[E] : 1.0f - f.s[E]) * (ch ? f.s[H] : 1.0f - f.s[H]);
            const int k0 = (ce << E) | (ch << H), k1 = k0 | (1 << D);
            a.x = fmaf(w, v[k1].x - v[k0].x, a.x);
            a.y = fmaf(w, v[k1].y - v[k0].y, a.y);
        }
    return a;
}

// B_de of both features (D != E): sum over the third dim of omega*(v_11 - v_10 - v_01 + v_00)
template <int D, int E>
__host__ __device__ __forceinline__ float2 diff_cross(const LevelFrame& f, const float2 (&v)[8])
{
    constexpr int H = 3 - D - E;
    float2 b = make_float2(0.f, 0.f);
#pragma unroll
    for (int ch = 0; ch < 2; ++ch) {
        const float w = ch ? f.s[H] : 1.0f - f.s[H];
        const int k00 = ch << H, k10 = k00 | (1 << D), k01 = k00 | (1 << E), k11 = k10 | (1 << E);
        b.x = fmaf(w, (v[k11].x - v[k10].x) - (v[k01].x - v[k00].x), b.x);
        b.y = fmaf(w, (v[k11].y - v[k10].y) - (v[k01].y - v[k00].y), b.y);
    }
    return b;
}

// acc_d += sum_f gl_f * dy_f/dx_d over one level: gl = dL/dy of the level's two features, v = its eight corner entries.
// The same three lines as encoding_grad.cu::bwd_input_sample, which keeps its own copy (calling this one there changed
// that kernel's register allocation).
__host__ __device__ __forceinline__ void level_input_grad(const LevelFrame& f, const float2 (&v)[8], float2 gl, float (&acc)[3])
{
    const float2 a0 = diff_along<0>(f, v), a1 = diff_along<1>(f, v), a2 = diff_along<2>(f, v);
    acc[0] = fmaf(f.scale * f.ds[0], fmaf(gl.x, a0.x, gl.y * a0.y), acc[0]);
    acc[1] = fmaf(f.scale * f.ds[1], fmaf(gl.x, a1.x, gl.y * a1.y), acc[1]);
    acc[2] = fmaf(f.scale * f.ds[2], fmaf(gl.x, a2.x, gl.y * a2.y), acc[2]);
}

}  // namespace perf
