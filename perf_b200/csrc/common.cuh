// common.cuh -- shared host/device helpers of libperfb200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <math.h>
#include <string.h>
#include "../../include/perfb200.h"

namespace perf {

// ---------------------------------------------------------------- errors
void set_error(const char* fmt, ...);
#define PERF_CHECK_ARG(cond, ...)  do { if (!(cond)) { perf::set_error(__VA_ARGS__); return PERF_EINVAL; } } while (0)
#define PERF_CHECK_SUP(cond, ...)  do { if (!(cond)) { perf::set_error(__VA_ARGS__); return PERF_EUNSUPPORTED; } } while (0)
#define PERF_CUDA(expr) do { cudaError_t e_ = (expr); if (e_ != cudaSuccess) { \
    perf::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e_), __FILE__, __LINE__); return PERF_ECUDA; } } while (0)
#define PERF_LAUNCH_CHECK() PERF_CUDA(cudaGetLastError())

int num_sms();   // cached multiprocessor count of the current device

// ---------------------------------------------------------------- grid level table
// Passed BY VALUE as a kernel parameter (272 bytes) -> lives in the constant bank.
struct LevelTable {
    float    scale[PERF_MAX_LEVELS];
    uint32_t res[PERF_MAX_LEVELS];
    uint32_t size[PERF_MAX_LEVELS];
    uint32_t offset[PERF_MAX_LEVELS];
    uint32_t n_levels;
    uint32_t hashed_mask;      // bit l set: level l is hashed
    uint32_t pow2_mask;        // bit l set: size[l] is a power of two (mod == and)
    uint32_t smoothstep;
};
int build_level_table(const perf_grid_cfg* cfg, LevelTable* out, uint64_t* n_entries);

// Layout of the packed gather table (perf_pack_tables): entries [0, n_entries) in parameter order, then a CELL-MAJOR copy
// of the leading dense levels -- for level l, res_l^3 cells x 8 corners x 8 bytes, cell (gx,gy,gz) at gx + res (gy + res gz),
// corner k (bit0 = x, bit1 = y, bit2 = z) holding entry ((gx+kx) + res (gy+ky) + res^2 (gz+kz)) % size of that level.
// The fused field kernels read a dense level as ONE 64-byte record per sample (4 x LDG.128, one address, no wrap test)
// instead of eight 8-byte gathers.  cell_start[l]: first entry (8-byte units) of level l's cells.
constexpr uint32_t PERF_CELL_LEVELS = 4;                 // PeRF's grid: levels 0..3 are dense
constexpr uint64_t PERF_CELL_CAP = 1ull << 20;           // at most 2^20 cells (64 MB) are ever duplicated
struct PackedLayout {
    uint32_t n_cell_levels;                              // leading dense levels with a cell-major copy (<= PERF_CELL_LEVELS)
    uint64_t cell_start[PERF_CELL_LEVELS];
    uint64_t total_entries;                              // n_entries + 8 * cells
};
inline PackedLayout packed_layout(const LevelTable& lt, uint64_t n_entries)
{
    PackedLayout pl; pl.n_cell_levels = 0; pl.total_entries = n_entries;
    uint64_t cells = 0;
    for (uint32_t l = 0; l < lt.n_levels && l < PERF_CELL_LEVELS; ++l) {
        if ((lt.hashed_mask >> l) & 1u) break;
        const uint64_t c = (uint64_t)lt.res[l] * lt.res[l] * lt.res[l];
        if (cells + c > PERF_CELL_CAP) break;
        pl.cell_start[l] = pl.total_entries; pl.total_entries += 8 * c; cells += c; pl.n_cell_levels = l + 1;
    }
    return pl;
}
int mlp_param_count(const perf_mlp_cfg* mlp, uint64_t* count);
int check_mlp(const perf_mlp_cfg* mlp);

#ifdef __CUDACC__
// ---------------------------------------------------------------- device: hash-grid addressing
// tcnn pos_fract / grid_index / coherent-prime hash (SURVEY.md Appendix A); mirrored 1:1 by
// oracle/hashgrid.py so that indices are bit-identical and the fp32 blend matches to the ulp.
struct Corner8 {
    uint32_t idx[8];     // absolute entry index (level offset included)
    float    w[8];       // trilinear weight, corner c: bit0=x, bit1=y, bit2=z
};

__host__ __device__ __forceinline__ uint32_t level_index(uint32_t gx, uint32_t gy, uint32_t gz,
                                                bool hashed, bool pow2, uint32_t res, uint32_t size)
{
    uint32_t idx;
    if (hashed) {
        idx = gx ^ (gy * 2654435761u) ^ (gz * 805459861u);
        idx = pow2 ? (idx & (size - 1u)) : (idx % size);
    } else {
        // dense stride walk; for these levels res^3 (rounded up to 8) == size so all three
        // dims participate.  (tcnn stops early only when stride > size, which implies hashed.)
        idx = gx + gy * res + gz * res * res;
        if (idx >= size) idx %= size;
    }
    return idx;
}

// round-to-nearest multiply that the compiler may not contract into an fma (device); plain IEEE multiply
// when the same source is compiled for the host by tests/host_harness.py
#ifdef __CUDA_ARCH__
#define PERF_FMUL_RN(a, b) __fmul_rn((a), (b))
#define PERF_FADD_RN(a, b) __fadd_rn((a), (b))
#define PERF_FSUB_RN(a, b) __fsub_rn((a), (b))
#define PERF_FDIV_RN(a, b) __fdiv_rn((a), (b))
#else
#define PERF_FMUL_RN(a, b) ((a) * (b))
#define PERF_FADD_RN(a, b) ((a) + (b))
#define PERF_FSUB_RN(a, b) ((a) - (b))
#define PERF_FDIV_RN(a, b) ((a) / (b))
#endif

// A level's cell frame at (x, y, z) (tcnn pos_fract): per axis pos = scale x + 0.5, g = its integer cell, p = fract(pos).
// The interpolation weights and corner indices built on it stay with each caller.
__host__ __device__ __forceinline__ void cell_frame(float scale, float x, float y, float z,
                                                    uint32_t& gx, uint32_t& gy, uint32_t& gz, float& px, float& py, float& pz)
{
    const float sx = fmaf(scale, x, 0.5f), sy = fmaf(scale, y, 0.5f), sz = fmaf(scale, z, 0.5f);
    const float fx = floorf(sx), fy = floorf(sy), fz = floorf(sz);
    gx = (uint32_t)(int)fx; gy = (uint32_t)(int)fy; gz = (uint32_t)(int)fz;
    px = sx - fx; py = sy - fy; pz = sz - fz;
}

__host__ __device__ __forceinline__ void level_corners(const LevelTable& lt, int l, float x, float y, float z, Corner8& c)
{
    const float scale = lt.scale[l];
    const uint32_t res = lt.res[l], size = lt.size[l], off = lt.offset[l];
    const bool hashed = (lt.hashed_mask >> l) & 1u, pow2 = (lt.pow2_mask >> l) & 1u;
    uint32_t gx, gy, gz; float wx, wy, wz;
    cell_frame(scale, x, y, z, gx, gy, gz, wx, wy, wz);
    if (lt.smoothstep) {
        wx = wx * wx * (3.0f - 2.0f * wx); wy = wy * wy * (3.0f - 2.0f * wy); wz = wz * wz * (3.0f - 2.0f * wz);
    }
    const float ox = 1.0f - wx, oy = 1.0f - wy, oz = 1.0f - wz;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        // weight = ((1 * ax) * ay) * az in this order (oracle/hashgrid.py::_corner_weights_indices)
        float w = PERF_FMUL_RN(PERF_FMUL_RN((k & 1) ? wx : ox, (k & 2) ? wy : oy), (k & 4) ? wz : oz);
        c.w[k] = w;
        c.idx[k] = off + level_index(gx + (k & 1), gy + ((k >> 1) & 1), gz + ((k >> 2) & 1), hashed, pow2, res, size);
    }
}

// Specialised addressing for the hot kernels: the level kind is a compile-time constant
// (HASHED levels must have a power-of-two size, dense levels use idx < 2*size), coordinates must
// lie in [0,1] (callers clamp masked-out samples) and interpolation is Linear.  Produces exactly
// the indices / weights of level_corners() under those preconditions -- no divisions, no branches.
template <bool HASHED>
__host__ __device__ __forceinline__ void level_corners_fast(const LevelTable& lt, int l, float x, float y, float z, Corner8& c)
{
    const float scale = lt.scale[l];
    const uint32_t res = lt.res[l], size = lt.size[l], off = lt.offset[l];
    uint32_t gx, gy, gz; float wx, wy, wz;
    cell_frame(scale, x, y, z, gx, gy, gz, wx, wy, wz);
    const float ox = 1.0f - wx, oy = 1.0f - wy, oz = 1.0f - wz;
    const float wxy[4] = {PERF_FMUL_RN(ox, oy), PERF_FMUL_RN(wx, oy), PERF_FMUL_RN(ox, wy), PERF_FMUL_RN(wx, wy)};
#pragma unroll
    for (int k = 0; k < 8; ++k) c.w[k] = PERF_FMUL_RN(wxy[k & 3], (k & 4) ? wz : oz);
    if constexpr (HASHED) {
        const uint32_t mask = size - 1u;
        const uint32_t hy0 = gy * 2654435761u, hy1 = hy0 + 2654435761u;
        const uint32_t hz0 = gz * 805459861u,  hz1 = hz0 + 805459861u;
        const uint32_t hyz[4] = {hy0 ^ hz0, hy1 ^ hz0, hy0 ^ hz1, hy1 ^ hz1};
        const uint32_t gx1 = gx + 1u;
#pragma unroll
        for (int k = 0; k < 8; ++k) c.idx[k] = off + ((((k & 1) ? gx1 : gx) ^ hyz[k >> 1]) & mask);
    } else {
        const uint32_t r2 = res * res;
        const uint32_t b00 = gx + gy * res + gz * r2;
        const uint32_t base[4] = {b00, b00 + res, b00 + r2, b00 + res + r2};
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            uint32_t i = base[k >> 1] + (uint32_t)(k & 1);
            i = (i >= size) ? i - size : i;                 // == i % size for i < 2*size
            c.idx[k] = off + i;
        }
    }
}
// Opaque bit operations (device: inline PTX the optimiser cannot re-associate; host harness: plain C).
// (a ^ b ^ c) & m is what the compiler makes of the hashed index -- per corner one 3-input XOR, one AND and one ADD of
// the level offset.  Masking the x term and the four (y ^ z) terms ONCE per level leaves a single 2-input XOR per corner.
__host__ __device__ __forceinline__ uint32_t xor_and_u32(uint32_t a, uint32_t b, uint32_t m)
{
#ifdef __CUDA_ARCH__
    uint32_t r; asm("lop3.b32 %0, %1, %2, %3, 0x28;" : "=r"(r) : "r"(a), "r"(b), "r"(m)); return r;     // (a ^ b) & m
#else
    return (a ^ b) & m;
#endif
}
__host__ __device__ __forceinline__ uint32_t and_u32(uint32_t a, uint32_t m)
{
#ifdef __CUDA_ARCH__
    uint32_t r; asm("and.b32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(m)); return r;
#else
    return a & m;
#endif
}

// level_corners_fast() with indices RELATIVE to the level's first entry: the caller adds lt.offset[l] to the table
// pointer once per level (idx_fast[k] == lt.offset[l] + idx[k], weights identical; tests/test_addressing_host.py).
// Hashed levels: 4 + 2 masked terms and one XOR per corner (see xor_and_u32).  Dense levels: the `% size` wrap can
// only trigger in cells on the far faces of the box, so ONE comparison per level guards the eight per-corner wraps.
template <bool HASHED>
__host__ __device__ __forceinline__ void level_corners_rel(const LevelTable& lt, int l, float x, float y, float z, uint32_t (&idx)[8], float (&w)[8])
{
    const float scale = lt.scale[l];
    const uint32_t res = lt.res[l], size = lt.size[l];
    uint32_t gx, gy, gz; float wx, wy, wz;
    cell_frame(scale, x, y, z, gx, gy, gz, wx, wy, wz);
    const float ox = 1.0f - wx, oy = 1.0f - wy, oz = 1.0f - wz;
    const float wxy[4] = {PERF_FMUL_RN(ox, oy), PERF_FMUL_RN(wx, oy), PERF_FMUL_RN(ox, wy), PERF_FMUL_RN(wx, wy)};
#pragma unroll
    for (int k = 0; k < 8; ++k) w[k] = PERF_FMUL_RN(wxy[k & 3], (k & 4) ? wz : oz);
    if constexpr (HASHED) {
        const uint32_t mask = size - 1u;
        const uint32_t hy0 = gy * 2654435761u, hy1 = hy0 + 2654435761u;
        const uint32_t hz0 = gz * 805459861u,  hz1 = hz0 + 805459861u;
        const uint32_t hyz[4] = {xor_and_u32(hy0, hz0, mask), xor_and_u32(hy1, hz0, mask), xor_and_u32(hy0, hz1, mask), xor_and_u32(hy1, hz1, mask)};
        const uint32_t hx[2] = {and_u32(gx, mask), and_u32(gx + 1u, mask)};
#pragma unroll
        for (int k = 0; k < 8; ++k) idx[k] = hx[k & 1] ^ hyz[k >> 1];
    } else {
        const uint32_t r2 = res * res;
        const uint32_t b00 = gx + gy * res + gz * r2;
        const uint32_t base[4] = {b00, b00 + res, b00 + r2, b00 + res + r2};
#pragma unroll
        for (int k = 0; k < 8; ++k) idx[k] = base[k >> 1] + (uint32_t)(k & 1);
        if (base[3] + 1u >= size) {                             // the largest of the eight; every index is < 2*size
#pragma unroll
            for (int k = 0; k < 8; ++k) idx[k] = (idx[k] >= size) ? idx[k] - size : idx[k];
        }
    }
}
// Dense level of the fused field kernels: cell index into the cell-major copy (PackedLayout) + the eight weights of
// level_corners_fast().  Coordinates in [0,1] => gx, gy, gz <= res - 1, i.e. cell < res^3.
__host__ __device__ __forceinline__ uint32_t level_cell_dense(const LevelTable& lt, int l, float x, float y, float z, float (&w)[8])
{
    const float scale = lt.scale[l];
    const uint32_t res = lt.res[l];
    uint32_t gx, gy, gz; float wx, wy, wz;
    cell_frame(scale, x, y, z, gx, gy, gz, wx, wy, wz);
    const float ox = 1.0f - wx, oy = 1.0f - wy, oz = 1.0f - wz;
    const float wxy[4] = {PERF_FMUL_RN(ox, oy), PERF_FMUL_RN(wx, oy), PERF_FMUL_RN(ox, wy), PERF_FMUL_RN(wx, wy)};
#pragma unroll
    for (int k = 0; k < 8; ++k) w[k] = PERF_FMUL_RN(wxy[k & 3], (k & 4) ? wz : oz);
    return gx + res * (gy + res * gz);
}

// host-side precondition of the fast path: `n_dense` leading dense levels, every other level
// hashed with a power-of-two size, Linear interpolation
inline bool fast_addressing_ok(const LevelTable& lt, uint32_t n_dense)
{
    if (lt.smoothstep) return false;
    for (uint32_t l = 0; l < lt.n_levels; ++l) {
        const bool hashed = (lt.hashed_mask >> l) & 1u, pow2 = (lt.pow2_mask >> l) & 1u;
        if (l < n_dense ? hashed : !(hashed && pow2)) return false;
    }
    return true;
}

// Scatter of one level's 8 corner contributions (float2 each) into an fp32 gradient table.
// V4: the two x-neighbours of a corner pair sit in the same 16-byte slot whenever their indices differ in bit 0
// only (always for a hashed level when the cell's x coordinate is even, and for a dense level when the index
// is even): one 16-byte vector atomic then replaces two 8-byte ones.  `dtable` must be 16-byte aligned for V4.
// (Host compilation = tests/host_harness.py: plain adds, one thread.)
__host__ __device__ __forceinline__ void grad_add2(float2* p, float2 v)
{
#ifdef __CUDA_ARCH__
    atomicAdd(p, v);
#else
    p->x += v.x; p->y += v.y;
#endif
}
__host__ __device__ __forceinline__ void grad_add4(float4* p, float4 v)
{
#ifdef __CUDA_ARCH__
    atomicAdd(p, v);
#else
    p->x += v.x; p->y += v.y; p->z += v.z; p->w += v.w;
#endif
}
template <bool V4>
__host__ __device__ __forceinline__ void scatter8(float2* __restrict__ dtable, const uint32_t (&idx)[8], const float2 (&v)[8])
{
#pragma unroll
    for (int k = 0; k < 8; k += 2) {
        const uint32_t i0 = idx[k], i1 = idx[k + 1];
        if (V4 && ((i0 ^ i1) == 1u)) {
            const bool swap = (i0 & 1u) != 0u;
            const float2 lo = swap ? v[k + 1] : v[k], hi = swap ? v[k] : v[k + 1];
            grad_add4(reinterpret_cast<float4*>(dtable + (i0 & ~1u)), make_float4(lo.x, lo.y, hi.x, hi.y));
        } else {
            grad_add2(dtable + i0, v[k]);
            grad_add2(dtable + i1, v[k + 1]);
        }
    }
}

__host__ __device__ __forceinline__ uint32_t pack_half2(float a, float b)
{
    __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
}
__host__ __device__ __forceinline__ float2 unpack_half2(uint32_t u)
{
    return __half22float2(*reinterpret_cast<__half2*>(&u));
}
__device__ __forceinline__ float round_half(float v) { return __half2float(__float2half_rn(v)); }

// Trilinear blend of one level, exactly as tcnn's kernel_grid does it for __half parameters:
// result = fma((half)weight_k, value_k, result) for corners k = 0..7, one fp16 rounding per fma
// (HFMA2 on the feature pair), starting from zero.  Mirrored by oracle/hashgrid.py::encode(blend="half").
__device__ __forceinline__ uint32_t blend8_half(const float (&w)[8], const uint32_t (&v)[8])
{
    __half2 acc = __float2half2_rn(0.f);
#pragma unroll
    for (int k = 0; k < 8; ++k) acc = __hfma2(__float2half2_rn(w[k]), *reinterpret_cast<const __half2*>(&v[k]), acc);
    return *reinterpret_cast<uint32_t*>(&acc);
}

// (p - lo) / ext, correctly rounded, for a divisor that is the same for every sample of the launch: with r = RN(1 / ext)
// computed once, q = RN(n r), q' = RN(q + RN(n - q ext) r) is the correctly rounded quotient (Markstein: the remainder is
// exact in one FMA; holds unless the significand of ext is all ones, which the host checks with div_uniform_ok) -- 3
// dependent FMA-pipe instructions per coordinate instead of the ~10 of the generic IEEE division (MUFU.RCP, refinement,
// range check).  __host__ __device__: tests/test_addressing_host.py compares the sequence with the IEEE division on the CPU.
#ifndef PERF_OPT_DIV
#define PERF_OPT_DIV 1
#endif
__host__ __device__ __forceinline__ float div_uniform(float n, float ext, float r, bool generic)
{
#if PERF_OPT_DIV
    if (generic) return PERF_FDIV_RN(n, ext);             // uniform branch; never taken for PeRF's [-1,1]^3 box
    const float q = PERF_FMUL_RN(n, r);
    return fmaf(fmaf(-q, ext, n), r, q);
#else
    (void)r; (void)generic; return PERF_FDIV_RN(n, ext);
#endif
}
// host-side precondition of the 3-FMA path: a normal-range extent whose significand is not all ones
inline bool div_uniform_ok(float ext)
{
    uint32_t bits; memcpy(&bits, &ext, 4);
    return (bits & 0x7FFFFFu) != 0x7FFFFFu && ext > 1e-30f && ext < 1e30f;
}

// ---------------------------------------------------------------- device: rays and sample positions (oracle/sampler.py)
// The backward kernels do not save sample positions: they recompute them from the rays with these helpers and must reach
// the forward's fp32 x01 bit for bit, or the gradients land in other cells.
// Fixed-S sampling: sample k of a ray covers [fixed_s_t(k), fixed_s_t(k + 1)), t(k) = near + (k + jit) step with
// step = (far - near) / S.
__host__ __device__ __forceinline__ float fixed_s_step(float near, float far, uint32_t S) { return PERF_FDIV_RN(PERF_FSUB_RN(far, near), (float)S); }
__host__ __device__ __forceinline__ float fixed_s_t(float near, float step, uint32_t k, float jit)
{
    return PERF_FADD_RN(near, PERF_FMUL_RN(PERF_FADD_RN((float)k, jit), step));
}
// One axis of the sample midpoint o + d (ts + te) / 2, with tsum = ts + te (ngp_nerf.py:137-140)
__host__ __device__ __forceinline__ float sample_midpoint(float o, float d, float tsum) { return PERF_FADD_RN(o, PERF_FMUL_RN(d, tsum) * 0.5f); }
// One axis of the box [lo, lo + ext] mapped to [0, 1].  The forward field kernels divide with div_uniform() instead (same
// subtraction): both divisions round correctly, so they agree bit for bit whenever div_uniform_ok() holds for every extent
// (otherwise div_uniform() takes this division itself), and the backward relies on that.
__host__ __device__ __forceinline__ float to_unit(float p, float lo, float ext) { return PERF_FDIV_RN(PERF_FSUB_RN(p, lo), ext); }

// torch.linspace(start, end, n)[i] in fp32 (ATen's symmetric formula), so that pixel centres match
// utils/camera_utils.py:113-117 to the ulp.
__host__ __device__ __forceinline__ float linspace(float start, float end, int i, int n)
{
    if (n == 1) return start;
    const float step = (end - start) / (float)(n - 1);
    return (i < n / 2) ? PERF_FADD_RN(start, PERF_FMUL_RN(step, (float)i)) : PERF_FSUB_RN(end, PERF_FMUL_RN(step, (float)(n - i - 1)));
}
// pixel-centre coordinate of pixel i of n in (0, 1)
__host__ __device__ __forceinline__ float linspace_val(int i, int n)
{
    return linspace((float)(0.5 / (double)n), (float)(1.0 - 0.5 / (double)n), i, n);
}
// camera-space equirect direction of pixel (row, col): camera_utils.py:120-126,142-147
__host__ __device__ __forceinline__ void pano_dir(int row, int col, int H, int W, float& dx, float& dy, float& dz)
{
    const float y = linspace_val(row, H), x = linspace_val(col, W);
    const float beta = -(y - 0.5f) * 3.14159274101257324f;            // float32(np.pi)
    const float alpha = -(x - 0.5f) * 6.28318548202514648f;           // float32(2 np.pi)
    float sa, ca, sb, cb;
    sincosf(alpha, &sa, &ca); sincosf(beta, &sb, &cb);
    dx = ca * cb; dy = sa * cb; dz = sb;
}
// apply_rot (camera_utils.py:44-46): d_world = R c, R row-major 3x3
__host__ __device__ __forceinline__ void rotate(const float (&r)[9], float cx, float cy, float cz, float& dx, float& dy, float& dz)
{
    dx = r[0] * cx + r[1] * cy + r[2] * cz;
    dy = r[3] * cx + r[4] * cy + r[5] * cz;
    dz = r[6] * cx + r[7] * cy + r[8] * cz;
}

// ---------------------------------------------------------------- device: wgmma / mbarrier PTX
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// Spin on an mbarrier phase with a bounded number of polls; a kernel that would hang traps
// instead (so a lost bulk-copy completion surfaces as a CUDA error, not a wedged GPU).
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity)
{
    const uint32_t addr = smem_u32(bar);
    uint32_t done = 0;
    long long t0 = 0;
    for (uint32_t spin = 0;; ++spin) {
        asm volatile("{\n\t.reg .pred p;\n\t"
                     "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
                     "selp.u32 %0, 1, 0, p;\n\t}"
                     : "=r"(done) : "r"(addr), "r"(parity) : "memory");
        if (done) return;
        if (spin == 64) t0 = clock64();
        if (spin > 64 && clock64() - t0 > 4000000000ll) __trap();    // ~2 s at 2 GHz
    }
}

// Shared-memory matrix descriptor of wgmma, no swizzle ("interleave"): 8 x 16-byte core matrices.
// K-major operand: LBO = byte distance between the two core matrices of one K=16 step, SBO = between 8-row groups.
// MN-major operand: LBO = byte distance between 8-row K groups, SBO = between 8-element MN groups.
__device__ __forceinline__ uint64_t gmma_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes)
{
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr >> 4) & 0x3FFFu);
    d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16;
    d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32;
    return d;                                     // base_offset 0, layout type 0 = no swizzle
}
__device__ __forceinline__ void wgmma_fence()  { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait()   { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }

// D[64 x N] (registers, fp32) (+)= A[64 x 16] * B[N x 16]^T, fp16 operands from shared memory; one warpgroup.
// TA / TB: the operand is MN-major (transposed).  Thread l of warp w holds rows 16w + l/4 (+8) and columns
// 8j + 2(l%4) (+1): d[4j] (row, col), d[4j+1] (row, col+1), d[4j+2] (row+8, col), d[4j+3] (row+8, col+1).
template <int TA, int TB>
__device__ __forceinline__ void wgmma_n64(float (&d)[32], uint64_t adesc, uint64_t bdesc, uint32_t accumulate)
{
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
                 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
                 "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
                 "%32, %33, p, 1, 1, %35, %36;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
                   "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
                   "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
                   "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
                 : "l"(adesc), "l"(bdesc), "r"(accumulate), "n"(TA), "n"(TB));
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_n32(float (&d)[16], uint64_t adesc, uint64_t bdesc, uint32_t accumulate)
{
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 "
                 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
                 "%16, %17, p, 1, 1, %19, %20;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
                   "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
                 : "l"(adesc), "l"(bdesc), "r"(accumulate), "n"(TA), "n"(TB));
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_n8(float (&d)[4], uint64_t adesc, uint64_t bdesc, uint32_t accumulate)
{
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %6, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n8k16.f32.f16.f16 "
                 "{%0, %1, %2, %3}, %4, %5, p, 1, 1, %7, %8;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "l"(adesc), "l"(bdesc), "r"(accumulate), "n"(TA), "n"(TB));
}

// The same with A from REGISTERS (K-major, fp16 pairs): thread l of warp w holds a[0] = (row 16w + l/4, cols 2(l%4), +1),
// a[1] = (row + 8, same cols), a[2] = (row, cols 8 + 2(l%4), +1), a[3] = (row + 8, cols 8 + 2(l%4), +1) -- the layout of
// accumulator pairs (4j, 4j+1), (4j+2, 4j+3) of two neighbouring column groups j of an m64nN fp32 fragment (relu_frag).
__device__ __forceinline__ void wgmma_n64_ra(float (&d)[32], const uint32_t* a, uint64_t bdesc, uint32_t accumulate)
{
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
                 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
                 "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
                 "{%32, %33, %34, %35}, %36, p, 1, 1, 0;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
                   "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
                   "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
                   "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_n8_ra(float (&d)[4], const uint32_t* a, uint64_t bdesc, uint32_t accumulate)
{
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %9, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n8k16.f32.f16.f16 "
                 "{%0, %1, %2, %3}, {%4, %5, %6, %7}, %8, p, 1, 1, 0;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(accumulate));
}
// m64n32k16 with A from registers and B MN-major (transposed): a data-gradient product against a forward weight image
__device__ __forceinline__ void wgmma_n32_ra_tb(float (&d)[16], const uint32_t* a, uint64_t bdesc, uint32_t accumulate)
{
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %21, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 "
                 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
                 "{%16, %17, %18, %19}, %20, p, 1, 1, 1;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
                   "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(accumulate));
}

// ---------------------------------------------------------------- byte streams (png.cu, jpeg.cu, h264.cu)
// Device: an atomic OR; host (the encoders' test harness builds and host-side writers): a plain one.
__host__ __device__ __forceinline__ void or_u32(uint32_t* p, uint32_t v)
{
#ifdef __CUDA_ARCH__
    atomicOr(p, v);
#else
    *p |= v;
#endif
}
__host__ __device__ __forceinline__ uint32_t bswap_u32(uint32_t v)
{
#ifdef __CUDA_ARCH__
    return __byte_perm(v, 0, 0x0123);
#else
    return __builtin_bswap32(v);
#endif
}
// The bits v takes, 0 for 0
__host__ __device__ __forceinline__ int bit_width(uint32_t v)
{
#ifdef __CUDA_ARCH__
    return 32 - __clz((int)v);
#else
    return v ? 32 - __builtin_clz(v) : 0;
#endif
}

// Bit sinks of the MSB-first codes (JPEG, H.264): BitCount adds up lengths; MsbBits ORs the bits into words that are zero
// where it writes, through a word-aligned 64-bit accumulator, one OR per 32 bits.  The words are stored byte-swapped, so on
// a little-endian machine the buffer reads as bytes in stream order.  (Deflate is LSB-first: png.cu has its own writer.)
struct BitCount {
    uint32_t n = 0;
    __host__ __device__ __forceinline__ void put(uint32_t, int nb) { n += nb; }
};
struct MsbBits {
    uint32_t* out; int64_t base; uint64_t acc; int fill;
    __host__ __device__ __forceinline__ MsbBits(uint32_t* o, int64_t pos) : out(o), base(pos & ~(int64_t)31), acc(0), fill((int)(pos & 31)) {}
    // the low nb bits of v, 0 <= nb <= 32: shifted to the top of a word (the bits above them drop out), then to bit `fill`
    __host__ __device__ __forceinline__ void put(uint32_t v, int nb)
    {
        if (nb == 0) return;
        acc |= (uint64_t)(v << (32 - nb)) << (32 - fill);
        fill += nb;
        if (fill >= 32) {
            or_u32(out + (base >> 5), bswap_u32((uint32_t)(acc >> 32)));
            acc <<= 32; fill -= 32; base += 32;
        }
    }
    __host__ __device__ __forceinline__ void flush()
    {
        if (fill > 0) or_u32(out + (base >> 5), bswap_u32((uint32_t)(acc >> 32)));
    }
    __host__ __device__ __forceinline__ int64_t pos() const { return base + fill; }     // the next bit's position
};

// Thread t's share [lo, hi) of n items over NT threads: contiguous runs of ceil(n / NT), the last ones short or empty.
template <class I> struct ItemRange { I lo, hi; };
template <int NT, class I>
__host__ __device__ __forceinline__ ItemRange<I> thread_range(I n, int t)
{
    const I q = (n + NT - 1) / NT;
    return {q * t < n ? q * t : n, q * (t + 1) < n ? q * (t + 1) : n};
}

// A CTA of NT threads that runs phases 0 .. NP - 1 of PHASE(args, shared state, CTA index, phase, thread) with a barrier
// after each.  The state is static shared memory when it fits the 48 KB static limit, dynamic shared memory otherwise.
constexpr size_t CTA_STATIC_SMEM = 48 * 1024;

template <class A, class S, int NT, int NP, void (*PHASE)(const A&, S&, int64_t, int, int)>
__global__ void __launch_bounds__(NT) cta_phases(const A a)
{
    S* s;
    if constexpr (sizeof(S) <= CTA_STATIC_SMEM) {
        __shared__ S static_smem;
        s = &static_smem;
    } else {
        extern __shared__ __align__(16) uint8_t dynamic_smem[];
        s = reinterpret_cast<S*>(dynamic_smem);
    }
    for (int p = 0; p < NP; ++p) {
        PHASE(a, *s, blockIdx.x, p, threadIdx.x);
        __syncthreads();
    }
}

// n_ctas CTAs of cta_phases on stream st; the host harness runs every thread of each phase of each CTA in a serial loop.
template <class A, class S, int NT, int NP, void (*PHASE)(const A&, S&, int64_t, int, int)>
int run_cta_phases(const A& a, int64_t n_ctas, cudaStream_t st)
{
#ifdef PERF_HOST_HARNESS
    (void)st;
    S* s = new S();
    for (int64_t c = 0; c < n_ctas; ++c)
        for (int p = 0; p < NP; ++p)
            for (int t = 0; t < NT; ++t) PHASE(a, *s, c, p, t);
    delete s;
#else
    constexpr size_t dyn = sizeof(S) <= CTA_STATIC_SMEM ? 0 : sizeof(S);
    if (dyn) PERF_CUDA(cudaFuncSetAttribute(cta_phases<A, S, NT, NP, PHASE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dyn));
    cta_phases<A, S, NT, NP, PHASE><<<(unsigned)n_ctas, NT, dyn, st>>>(a);
    PERF_LAUNCH_CHECK();
#endif
    return PERF_OK;
}
#endif  // __CUDACC__

}  // namespace perf
