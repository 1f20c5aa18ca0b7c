// render.cu -- the fused per-ray megakernel: ray-gen -> fixed-S sampling -> hash-grid encode of
// BOTH fields (hashed levels: one 8-byte gather per corner from the interleaved table; dense levels:
// one 64-byte cell record) -> density MLP and colour MLP on wgmma -> alpha composite (a running
// sum per thread in render_march_kernel, warp-shuffle segmented scans in the legacy render_kernel).
// Nothing per-sample ever touches HBM: inputs are the pose (or [R,3] rays) and the tables,
// outputs are 16-20 B per ray.
//
// Replaces the whole inner stack of SURVEY.md section 3.1:
//   NeRFScene.render / render_once      modules/scene/nerf.py:74-123
//   NeRFOCCRenderer.render              modules/scene/nerf_renderer.py:112-209 (fixed-S sampler)
//   NGPNeRF.query_density / query_rgb   modules/fields/ngp_nerf.py:136-162
//   gen_pano_rays                       utils/camera_utils.py:229-234
// Arithmetic contract: oracle/render.py::render_rays(mixed=True).
#include "mlp_tc.cuh"
#include "grid_grad.cuh"

namespace perf {

struct RenderArgs {
    LevelTable    lt;
    const uint2*  table;        // {geo half2, app half2} per entry
    const uint4*  cells[PERF_CELL_LEVELS];   // cell-major copies of the dense levels inside the same buffer (common.cuh::PackedLayout)
    const __half* geo_w;        // W1 [64,32] | Wout [16,64]
    const __half* app_w;        // W1 [64,32] | W2 [64,64] | Wout [16,64]
    float         aabb_min[3], aabb_ext[3];
    uint32_t      S;            // samples per ray
    uint32_t      rays_per_unit, tiles_per_unit;
    float         near, far;
    uint32_t      training;
    uint32_t      tile_mul;     // image-shaped work: tile = (i * tile_mul) % n_tiles (a bijection, gcd(tile_mul, n_tiles) == 1); 0 / 1 = row-major
    uint32_t      div_generic;  // 1: an aabb extent whose significand is all ones -> div_uniform() falls back to the IEEE division
    const float*  jitter;       // [R] or null
    const float*  bg_noise;     // [R,4] or null
    float*        rgb;          // [R,3]
    float*        distance;     // [R]
    float*        opacity;      // [R] or null
    uint64_t      R;
    // ray source
    const float*  rays_o;       // [R,3]  (PANO == false)
    const float*  rays_d;
    float         pose_r[9], pose_t[3];
    int           H, W, row0;   // (PANO == true): ray r is pixel (row0 + r / W, r % W)
    // packed variable-length samples (perf_render_packed): ray r owns samples [pk_offsets[r], pk_offsets[r+1])
    const int64_t* pk_offsets;  // [R+1] or null (fixed-S lattice)
    const float*   pk_ts;       // [N]
    const float*   pk_te;       // [N]
    // training-forward saves (SAVE != 0), all sample-major: row = k * R + ray
    float*        s_sigma;      // [S*R]
    float*        s_w;          // [S*R]
    float*        s_trans;      // [S*R]
    __half*       s_rgb;        // [S*R, 4] (colour phase only; 4th lane unused)
    uint4*        s_feat;       // [S*R, 32] fp16 of the network being trained
    uint4*        s_h1;         // [S*R, 64] fp16
    uint4*        s_h2;         // [S*R, 64] fp16 (colour phase only)
    float*        s_dacc;       // [R] distance accumulate BEFORE the background rule
    float*        s_dl;         // [R] distortion-loss numerator of the ray
    // ray splitting (explicit rays, fixed S): every ray is cut into `seg` consecutive segments of
    // S/seg samples handled by `seg` different threads of the tile (tile = 128/seg rays); the segment
    // results are combined with the transmittance product rule.  Fills the GPU for small ray batches
    // (an 8192-ray training batch is only 64 tiles of 128 rays, but 512 tiles of 16 rays x 8 segments).
    uint32_t      seg;          // power of two, divides S and 128; 1 = off
    union {
        float*    s_toff;       // [seg * R] transmittance at the start of each segment (SAVE, seg > 1)
        float*    normal;       // [R,3] sum_i w_i n_i per ray (NORMAL kernels: eval, seg == 1)
    };
};

// Shared memory of a field kernel = one CTA-wide block (the weight operand images, staged once per CTA, and the mbarrier
// of their bulk copy), then one region per warpgroup (WG_MAX of them at most, one 128-row tile each): the 4 tiles an SM
// runs at a time read ONE copy of the weights, and what shared memory they do not use is L1 for the table gathers.
// No warpgroup touches another warpgroup's region.
constexpr int WG_MAX = 4;
constexpr int align128(int b) { return (b + 127) / 128 * 128; }
constexpr int W_IMG_BYTES = W32_BYTES + W32_BYTES + W64_BYTES;       // 16 KB: W1 density | W1 colour | W2 colour
constexpr int WO_BYTES = 8 * HID * 2;               // 1 KB: an output layer as an N = 8 operand image (mlp_tc.cuh layout, LBO = 128)
constexpr int WO_LBO   = 8 * 16;
constexpr int W_IMG_ALL = W_IMG_BYTES + 2 * WO_BYTES;                // 18 KB: the hidden images, then the two output images
// measurement hook (tools/ab_lib.py): extra, unused dynamic shared memory per warpgroup of the field kernels, i.e. what
// more shared memory would cost in L1 capacity
#ifndef PERF_RS_PAD
#define PERF_RS_PAD 0
#endif

// Bytes the carveout percentage set_smem requests stands for on the H100 (228 KB of shared memory per SM at most): the
// driver takes the next supported carveout at or above it, so a layout meant for a given carveout must keep this under it.
constexpr long long carveout_request(long long need) { return (100 * need + 233471) / 233472 * 233472 / 100; }

// Shared-memory layout of a field kernel: byte offsets in the CTA-wide block, then in a warpgroup's region.
// EVAL: the eval kernels (wgmma MLP, no saves: eval_mlp_regs) keep the hidden layers in registers, so a warpgroup needs its
// feature tile only; the output layers are operand images too.  Otherwise the round trip: the training forward (SAVE = 1/2),
// the SIMT twin and the legacy scan kernel pass every hidden layer through shared memory.
// NORMAL (eval only): the normals kernels append per thread the sample position and the ray's running sum w n: the layer-1
// peak of the MLP leaves no register for them (the eval march kernel uses all 128 without them).
// L0SMEM (eval only, experiment PERF_FLAG_L0_SMEM): level 0 of the packed table (16^3 entries x 8 B = 32 KB) resident in
// shared memory behind the weights, staged once per persistent CTA by ONE bulk copy and read by all its warpgroups.
template <bool EVAL_, bool NORMAL_ = false, bool L0SMEM_ = false>
struct FieldLayout {
    static constexpr bool EVAL = EVAL_, NORMAL = NORMAL_, L0SMEM = L0SMEM_;
    static_assert(EVAL || (!NORMAL && !L0SMEM), "normals and level 0 in shared memory: eval layout only");
    // CTA-wide block: the weight operand images (W_BYTES, one bulk copy from g_wimg), the mbarrier of that copy (BARW);
    // L0SMEM: the mbarrier of the level-0 copy and level 0
    static constexpr int W1G = 0, W1A = W1G + W32_BYTES, W2A = W1A + W32_BYTES;
    static constexpr int WOG = W2A + W64_BYTES, WOA = WOG + WO_BYTES;        // EVAL: density row 0 / colour rows 0-2, the rest zero
    static constexpr int W_BYTES = EVAL ? W_IMG_ALL : W_IMG_BYTES, BARW = W1G + W_BYTES;
    static constexpr int BARL0 = align128(BARW + 16), L0 = BARL0 + 128, L0_BYTES = 4096 * 8;
    static constexpr int CTA = L0SMEM ? L0 + L0_BYTES : align128(BARW + 16);
    static_assert(W1A == W1G + W32_BYTES && W2A == W1A + W32_BYTES && WOG == W1G + W_IMG_BYTES && WOA == WOG + WO_BYTES,
                  "the weight images are one contiguous block, the layout of g_wimg");
    // per warpgroup: A = A_geo | A_app (16 KB; in the round trip later the colour hidden layers, K = 64); round trip: H = the
    // density hidden layer (16 KB), render_kernel's scan TAILS [2 scans][4 warps][8] and CARRY [2 parities][8] floats
    static constexpr int A = 0, H = A + A64_BYTES, TAILS = H + A64_BYTES, CARRY = TAILS + 2 * 4 * 8 * 4;
    // [4 warps] longest packed ray (perf_render_packed); the round trip aliases the tails: the scan kernel renders no packed rays
    static constexpr int MAX = EVAL ? A + A64_BYTES : TAILS;
    static constexpr int XYZ = MAX + 16, NACC = XYZ + TILE * 16;             // NORMAL: float4 [128] x01, selector; float [3][128] sum w n
    static constexpr int WG = align128(!EVAL ? CARRY + 2 * 8 * 4 : NORMAL ? NACC + 3 * TILE * 4 : MAX + 16);
    static constexpr int bytes(int nwg) { return CTA + nwg * (WG + PERF_RS_PAD); }   // the CTA-wide block, then nwg regions
};
// WG_MAX warpgroups of layout L take `total` bytes (PERF_RS_PAD aside), and with the 1 KB reserved per CTA they fit the
// `kb` KB carveout.  The four layouts, as DESIGN.md section 3 quotes them:
template <class L> constexpr bool layout_is(int total, int kb) { return L::CTA + WG_MAX * L::WG == total && carveout_request(total + 1024) <= kb * 1024; }
static_assert(layout_is<FieldLayout<true>>(18560 + 4 * 16512, 100), "eval layout: 84 608 B, the 100 KB carveout");
static_assert(layout_is<FieldLayout<true, true>>(18560 + 4 * 20096, 100), "normals layout: 98 944 B, the 100 KB carveout");
static_assert(layout_is<FieldLayout<false>>(16512 + 4 * 33152, 164), "round-trip layout: 149 120 B, the 164 KB carveout");
static_assert(layout_is<FieldLayout<true, false, true>>(117504, 132), "level-0 layout: 117 504 B, the 132 KB carveout");
// The layout of each field kernel, read by the kernel and by its launch (launch_march, launch_packed, launch_scan).
// render_march_kernel<PANO, SIMT, NDENSE, SAVE, L0SMEM, NORMAL> and packed_fields_kernel<NDENSE, SAVE, NORMAL> (SIMT = false):
// the eval layout unless the MLP runs on CUDA cores or saves.  render_kernel: the round trip.
template <bool SIMT, int SAVE, bool L0SMEM = false, bool NORMAL = false>
using MarchLayout = FieldLayout<!SIMT && SAVE == 0, NORMAL, L0SMEM>;
using ScanLayout = FieldLayout<false>;

// Output-layer weights of both networks as fp32 in the CONSTANT bank: [0,64) density row, [64,256) the three colour
// rows.  The 64 * n_out FMAs per sample of the output layers then take their weight operand straight from c[bank][imm]
// -- no load instruction (in shared memory they cost 64 broadcast LDS.128 per thread and sample on the L1 data pipe
// that bounds the kernel).  Filled from the fp16
// parameter vectors by weights_prepare_kernel, stream-ordered in front of every render launch (graph-capturable).
// One slot per device: renders of DIFFERENT fields on the same device must not overlap in time (different streams).
__constant__ float c_wout[4 * HID];
// The three hidden-layer matrices as ready-made wgmma operand images (no-swizzle K-major canonical layout, mlp_tc.cuh), 16 KB,
// followed by the two output layers as N = 8 operand images (2 x 1 KB, read by the eval kernels only): every persistent CTA
// stages them with ONE bulk copy (cp.async.bulk -> UBLKCP, completion on an mbarrier) instead of 1024+ 16-byte LDG + STS per
// CTA.  Written by the same preparation kernel, same single-slot rule as c_wout.
__device__ uint4 g_wimg[W_IMG_ALL / 16];

__global__ void __launch_bounds__(1024) weights_prepare_kernel(const __half* __restrict__ geo_w, const __half* __restrict__ app_w, float* __restrict__ c_dst)
{
    const int c = threadIdx.x;                       // 1024 threads = 1024 16-byte chunks of the hidden images
    if (c < 4 * HID) c_dst[c] = __half2float(c < HID ? geo_w[HID * 32 + c] : app_w[HID * 32 + HID * HID + (c - HID)]);
    const __half* src; int K, cc;
    if (c < 256)      { src = geo_w;            K = 32; cc = c; }
    else if (c < 512) { src = app_w;            K = 32; cc = c - 256; }
    else              { src = app_w + HID * 32; K = 64; cc = c - 512; }
    const int n = cc % HID, kg = cc / HID;           // image chunk (kg * 64 + n) <- row n, columns [8 kg, 8 kg + 8)
    g_wimg[c] = *reinterpret_cast<const uint4*>(src + (size_t)n * K + kg * 8);
    if (c < 2 * WO_BYTES / 16) {                     // output images: chunk (kg * 8 + n) <- output row n, columns [8 kg, 8 kg + 8)
        const int app = c >= WO_BYTES / 16, co = c % (WO_BYTES / 16), no = co % 8, kgo = co / 8;
        const __half* wout = app ? app_w + HID * 32 + HID * HID : geo_w + HID * 32;      // [16 (padded), 64]
        g_wimg[W_IMG_BYTES / 16 + c] = no < (app ? 3 : 1) ? *reinterpret_cast<const uint4*>(wout + no * HID + kgo * 8) : make_uint4(0, 0, 0, 0);
    }
}

// all threads of the CTA: weight images global -> the CTA-wide block of layout L by one bulk copy; returns when they have
// landed.  The eval layout takes all five images, the round trip the three hidden-layer ones.
template <class L>
__device__ __forceinline__ void stage_weights_bulk(uint8_t* smem)
{
    uint64_t* barw = reinterpret_cast<uint64_t*>(smem + L::BARW);
    if (threadIdx.x == 0) {
        mbar_init(barw, 1); fence_mbar_init();
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(smem_u32(barw)), "r"(L::W_BYTES) : "memory");
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                     :: "r"(smem_u32(smem + L::W1G)), "l"(reinterpret_cast<const void*>(g_wimg)), "r"(L::W_BYTES), "r"(smem_u32(barw)) : "memory");
    }
    __syncthreads();                                 // the barrier is initialised before anyone polls it
    mbar_wait(barw, 0);
}

// acc[o] += h[32C + 2j, 32C + 2j + 1] * c_wout[BASE + 64 o + 32 C + 2j, ... + 1]: even / odd partial sums, one fma2 per
// packed pair of activations (mlp_tc.cuh::out_dots has the same order); C is a compile-time constant so that the
// weights come straight from the constant bank (LDCU.128 of four weights into uniform registers).
template <int NOUT, int BASE, int C>
__device__ __forceinline__ void out_dots_const(const uint32_t (&p)[16], float2 (&acc)[NOUT])
{
#pragma unroll
    for (int j = 0; j < 16; ++j) {
        const float2 f = unpack_half2(p[j]);
#pragma unroll
        for (int o = 0; o < NOUT; ++o)
            fma2(acc[o], f, make_float2(c_wout[BASE + o * HID + 32 * C + 2 * j], c_wout[BASE + o * HID + 32 * C + 2 * j + 1]));
    }
}

// Inclusive scan of NV values along the ray across the whole CTA tile (and across the tiles of
// a unit through `carry`).  Lanes are consecutive samples; a ray may start anywhere.
//   k        : index of this sample inside its ray
//   k0_tile  : in-ray index of the tile's first sample (sample of thread 0)
// Deterministic: tree inside a warp, then warps in order, then tiles in order.
template <int NV>
__device__ __forceinline__ void ray_scan(float (&val)[NV], float (&excl)[NV], uint32_t k, uint32_t k0_tile, uint32_t S, int tid,
                                         float* tails /*[4][8]*/, const float* carry_in /*[8] or null*/, float* carry_out /*[8]*/)
{
    const int lane = tid & 31, warp = tid >> 5;
    const int seg_start = (k >= (uint32_t)lane) ? 0 : lane - (int)k;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
#pragma unroll
        for (int j = 0; j < NV; ++j) {
            const float t = __shfl_up_sync(0xffffffffu, val[j], off);
            if (lane - off >= seg_start) val[j] += t;
        }
    }
#pragma unroll
    for (int j = 0; j < NV; ++j) {               // exclusive prefix inside the warp (no inf - inf)
        const float t = __shfl_up_sync(0xffffffffu, val[j], 1);
        excl[j] = (lane - 1 >= seg_start) ? t : 0.f;
    }
    if (lane == 31) {
#pragma unroll
        for (int j = 0; j < NV; ++j) tails[warp * 8 + j] = val[j];
    }
    __syncthreads();
    // carry into the ray of lane 0 of warp w:  c[0] = carry_in;  c[w+1] = k0(w+1)==0 ? 0 : (one_seg(w) ? c[w] : 0) + tail[w]
    float c[NV];
#pragma unroll
    for (int j = 0; j < NV; ++j) c[j] = (carry_in != nullptr && k0_tile != 0) ? carry_in[j] : 0.f;
    const int upto = (carry_out != nullptr && tid == 0) ? 4 : warp;     // thread 0 also produces the tile's carry-out
    float cw[NV];
#pragma unroll
    for (int j = 0; j < NV; ++j) cw[j] = c[j];
#pragma unroll 1
    for (int w = 0; w < upto; ++w) {
        const uint32_t k0w = (k0_tile + 32u * w) % S;            // in-ray index of lane 0 of warp w
        const uint32_t k0n = (k0_tile + 32u * (w + 1)) % S;      // ... of lane 0 of warp w+1
        const bool one_seg = (k0w + 31u) < S;                    // warp w lies inside one ray
#pragma unroll
        for (int j = 0; j < NV; ++j) {
            const float prev = one_seg ? c[j] : 0.f;
            c[j] = (k0n == 0) ? 0.f : prev + tails[w * 8 + j];
        }
        if (w + 1 == warp) {
#pragma unroll
            for (int j = 0; j < NV; ++j) cw[j] = c[j];
        }
    }
    if (carry_out != nullptr && tid == 0) {
#pragma unroll
        for (int j = 0; j < NV; ++j) carry_out[j] = c[j];
    }
    if (k >= (uint32_t)lane) {               // same ray as lane 0 of my warp
#pragma unroll
        for (int j = 0; j < NV; ++j) { val[j] += cw[j]; excl[j] += cw[j]; }
    }
}

// Pixel-patch tiling of a 128-thread tile: a warp covers PATCH_WW x PATCH_WH pixels, the tile's four
// warps are arranged PATCH_WX x PATCH_WY.
#ifndef PATCH_WW
#define PATCH_WW 8
#define PATCH_WH 4
#define PATCH_WX 2
#define PATCH_WY 2
#endif
constexpr int PATCH_W = PATCH_WW * PATCH_WX, PATCH_H = PATCH_WH * PATCH_WY;
static_assert(PATCH_WW * PATCH_WH == 32 && PATCH_WX * PATCH_WY == 4, "a warp is 32 pixels, a tile 4 warps");

// Tiles of an image-shaped launch: patch_cols(W) across an image W pixels wide, patch_rows(rows) down one `rows` high.
__host__ __device__ __forceinline__ int patch_cols(int W) { return (W + PATCH_W - 1) / PATCH_W; }
__host__ __device__ __forceinline__ int patch_rows(int rows) { return (rows + PATCH_H - 1) / PATCH_H; }
// Pixel (prow, pcol) of lane `lane` of warp `warp` in patch tile `tile`, tiles_x = patch_cols(W) tiles per image row.
__device__ __forceinline__ void patch_pixel(uint64_t tile, uint32_t tiles_x, int warp, int lane, int& prow, int& pcol)
{
    const int ty = (int)(tile / tiles_x), tx = (int)(tile % tiles_x);
    prow = ty * PATCH_H + (warp / PATCH_WX) * PATCH_WH + lane / PATCH_WW;
    pcol = tx * PATCH_W + (warp % PATCH_WX) * PATCH_WW + lane % PATCH_WW;
}

struct RenderSmem {
    uint8_t *sA, *sAg, *sAa, *sH, *sW1g, *sW1a, *sW2a;
    uint8_t *sWog, *sWoa;   // output-layer operand images (eval layout), or null
    const uint2* l0;        // level 0 of the packed table in shared memory, or null
    float4* xyz;            // NORMAL kernels: [128] each thread's sample position + selector across the MLP, or null
};

// Warpgroup wg's view of a field kernel's shared memory in layout L (wg warp-uniform: see render_march_kernel): the
// RenderSmem, and the start of the warpgroup's region in `region` (not a member of RenderSmem: one there changes the SASS).
template <class L>
__device__ __forceinline__ RenderSmem field_smem(uint8_t* smem, int wg, uint8_t*& region)
{
    region = smem + (L::CTA + wg * L::WG) + wg * PERF_RS_PAD;
    uint8_t* const sA = region + L::A;
    return {sA, sA, sA + A32_BYTES, L::EVAL ? nullptr : region + L::H, smem + L::W1G, smem + L::W1A, smem + L::W2A,
            L::EVAL ? smem + L::WOG : nullptr, L::EVAL ? smem + L::WOA : nullptr,
            L::L0SMEM ? reinterpret_cast<const uint2*>(smem + L::L0) : nullptr,
            L::NORMAL ? reinterpret_cast<float4*>(region + L::XYZ) : nullptr};
}

// base + 8 * idx as ONE IMAD.WIDE.U32 (left to itself ptxas splits the 64-bit address into LEA + IADD3.X per corner)
__device__ __forceinline__ const uint2* entry_ptr(const uint2* base, uint32_t idx)
{
    uint64_t p;
    asm("mad.wide.u32 %0, %1, 8, %2;" : "=l"(p) : "r"(idx), "l"(reinterpret_cast<uint64_t>(base)));
    return reinterpret_cast<const uint2*>(p);
}

// L1 eviction hints of the table gathers.  The fine hashed levels stream through L1 (a ray leaves a fine cell with every
// step) while the dense / coarse levels are re-read from one sample to the next: 0 = default, 1 = L1::evict_first,
// 2 = L1::no_allocate, 3 = L1::evict_last.  (A/B: tools/ab_lib.py.)
#ifndef PERF_L1_HASHED
#define PERF_L1_HASHED 0
#endif
#ifndef PERF_L1_DENSE
#define PERF_L1_DENSE 0
#endif
template <int HINT>
__device__ __forceinline__ uint2 ldg_entry(const uint2* p)
{
    if constexpr (HINT == 0) return __ldg(p);
    uint2 v;
    if constexpr (HINT == 1) asm("ld.global.nc.L1::evict_first.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "l"(p));
    if constexpr (HINT == 2) asm("ld.global.nc.L1::no_allocate.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "l"(p));
    if constexpr (HINT == 3) asm("ld.global.nc.L1::evict_last.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "l"(p));
    return v;
}
template <int HINT>
__device__ __forceinline__ uint4 ldg_cell(const uint4* p)
{
    if constexpr (HINT == 0) return __ldg(p);
    uint4 v;
    if constexpr (HINT == 1) asm("ld.global.nc.L1::evict_first.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
    if constexpr (HINT == 2) asm("ld.global.nc.L1::no_allocate.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
    if constexpr (HINT == 3) asm("ld.global.nc.L1::evict_last.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
    return v;
}

// Levels [4q, 4q+4) of both fields -> one 16-byte k-group of row `row` of each feature tile.
// KIND 0: generic addressing, 1: dense (fast), 2: hashed power-of-two (fast).
template <int KIND, int SAVE, bool L0SMEM = false>
__device__ __forceinline__ void encode_group(const RenderArgs& a, const RenderSmem& sm, int q, float x, float y, float z, int row, uint64_t srow)
{
    uint32_t pg[4], pa[4];
#pragma unroll
    for (int ll = 0; ll < 4; ++ll) {
        const int l = 4 * q + ll;
        uint2 v[8]; float w[8];
        if constexpr (KIND == 0) {
            Corner8 c; level_corners(a.lt, l, x, y, z, c);
#pragma unroll
            for (int kk = 0; kk < 8; ++kk) { v[kk] = __ldg(a.table + c.idx[kk]); w[kk] = c.w[kk]; }
        } else if constexpr (KIND == 1) {
            if (L0SMEM && l == 0) {                // measured variant: level 0 (entry-major, offset 0) resident in shared memory
                uint32_t idx[8];
                level_corners_rel<false>(a.lt, l, x, y, z, idx, w);
#pragma unroll
                for (int kk = 0; kk < 8; ++kk) v[kk] = sm.l0[idx[kk]];
            } else {
                // dense level: ONE 64-byte cell record (all 8 corners of both fields), 4 x LDG.128 from one address
                const uint32_t cell = level_cell_dense(a.lt, l, x, y, z, w);
                const uint4* const cp = a.cells[l] + 4ull * cell;
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const uint4 c2 = ldg_cell<PERF_L1_DENSE>(cp + j);
                    v[2 * j] = make_uint2(c2.x, c2.y); v[2 * j + 1] = make_uint2(c2.z, c2.w);
                }
            }
        } else {
            // hashed level, level-local indices: the level offset goes into the pointer once, not into each of the 8 indices
            uint32_t idx[8];
            level_corners_rel<true>(a.lt, l, x, y, z, idx, w);
            const uint2* const tl = a.table + a.lt.offset[l];
#pragma unroll
            for (int kk = 0; kk < 8; ++kk) v[kk] = ldg_entry<PERF_L1_HASHED>(entry_ptr(tl, idx[kk]));
        }
        uint32_t vg[8], va[8];
#pragma unroll
        for (int kk = 0; kk < 8; ++kk) { vg[kk] = v[kk].x; va[kk] = v[kk].y; }
        pg[ll] = blend8_half(w, vg); pa[ll] = blend8_half(w, va);
    }
    *reinterpret_cast<uint4*>(sm.sAg + (q * TILE + row) * 16) = make_uint4(pg[0], pg[1], pg[2], pg[3]);
    *reinterpret_cast<uint4*>(sm.sAa + (q * TILE + row) * 16) = make_uint4(pa[0], pa[1], pa[2], pa[3]);
    if constexpr (SAVE == 1) { if (srow != ~0ull) a.s_feat[srow * 4 + q] = make_uint4(pg[0], pg[1], pg[2], pg[3]); }
    if constexpr (SAVE == 2) { if (srow != ~0ull) a.s_feat[srow * 4 + q] = make_uint4(pa[0], pa[1], pa[2], pa[3]); }
}

// Both MLPs of the eval kernels with every hidden layer in registers (the FlashAttention-3 treatment of P: an m64nN fp32
// accumulator fragment, ReLU-rounded pairwise to fp16, is the A-operand register fragment of the next m64nNk16 wgmma).
// Thread (warp w, lane l) owns row eval_row() = 64 (l / 16) + 16 w + l % 16 of the feature tiles: M = 64 half l / 16, and
// inside it rows [16w, 16w + 16) -- warp w's own slice of every fragment.  Per half h:
//   layer 1 of both nets, A = feature tile, B = W1 image            -> relu_frag -> hg, ha
//   colour layer 2 (A = ha, B = W2), density output (N = 8, A = hg)  -> relu_frag -> h2
//   colour output (N = 8, A = h2)
// Column c of in-warp row i of a half's N = 8 output is in lane 4 (i % 8) + c / 2, register 2 (i / 8) + c % 2, so every
// output of the row a thread owns is in a lane of its own warp: 16 shuffles, no barrier.  Returns the fp32 pre-activations.
// Shared memory is only read.  Before: the feature tiles are written, fenced for the async proxy and behind a barrier.  The
// barrier after the last layer-1 wgmma has completed lets the caller write the next tile.
__device__ __forceinline__ int eval_row(int tid) { return 64 * ((tid & 31) >> 4) + 16 * (tid >> 5) + (tid & 15); }

__device__ __forceinline__ void eval_mlp_regs(const RenderSmem& sm, int lane, float& lg, float& lr, float& lgr, float& lb)
{
    float os[2][4], oc[2][4];                               // N = 8 output fragments of both halves
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        uint32_t hg[16], ha[16];
        {
            float dg[32], da[32];
#pragma unroll
            for (int i = 0; i < 32; ++i) { dg[i] = 0.f; da[i] = 0.f; }
            wgmma_fence();
#pragma unroll
            for (int ks = 0; ks < 2; ++ks)
                wgmma_n64<0, 0>(dg, gmma_desc(smem_u32(sm.sAg) + h * 64 * 16 + ks * 2 * A_LBO, A_LBO, X_SBO),
                                gmma_desc(smem_u32(sm.sW1g) + ks * 2 * W_LBO, W_LBO, X_SBO), ks > 0 ? 1u : 0u);
#pragma unroll
            for (int ks = 0; ks < 2; ++ks)
                wgmma_n64<0, 0>(da, gmma_desc(smem_u32(sm.sAa) + h * 64 * 16 + ks * 2 * A_LBO, A_LBO, X_SBO),
                                gmma_desc(smem_u32(sm.sW1a) + ks * 2 * W_LBO, W_LBO, X_SBO), ks > 0 ? 1u : 0u);
            wgmma_commit();
            wgmma_wait();
            relu_frag(dg, hg);
            relu_frag(da, ha);
        }
        if (h == 1) wg_sync();                              // no warp reads the feature tiles any more
        float d2[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) d2[i] = 0.f;
#pragma unroll
        for (int i = 0; i < 4; ++i) { os[h][i] = 0.f; oc[h][i] = 0.f; }
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < 4; ++ks)
            wgmma_n64_ra(d2, ha + 4 * ks, gmma_desc(smem_u32(sm.sW2a) + ks * 2 * W_LBO, W_LBO, X_SBO), ks > 0 ? 1u : 0u);
#pragma unroll
        for (int ks = 0; ks < 4; ++ks)                      // N = 8: one 8-row group, SBO unused
            wgmma_n8_ra(os[h], hg + 4 * ks, gmma_desc(smem_u32(sm.sWog) + ks * 2 * WO_LBO, WO_LBO, X_SBO), ks > 0 ? 1u : 0u);
        wgmma_commit();
        wgmma_wait();
        uint32_t h2[16];
        relu_frag(d2, h2);
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < 4; ++ks)
            wgmma_n8_ra(oc[h], h2 + 4 * ks, gmma_desc(smem_u32(sm.sWoa) + ks * 2 * WO_LBO, WO_LBO, X_SBO), ks > 0 ? 1u : 0u);
        wgmma_commit();
        wgmma_wait();
    }
    // lane l wants column c of row l % 16 of half l / 16: register 2 ((l / 8) % 2) + c % 2 of half l / 16 in lane 4 (l % 8) + c / 2
    const int src = 4 * (lane & 7);
    const bool hi = (lane & 8) != 0, h1 = (lane & 16) != 0;
    auto fetch = [&](const float (&o)[2][4], int c, int from) {
        const float v0 = __shfl_sync(0xffffffffu, o[0][c], from), v1 = __shfl_sync(0xffffffffu, o[0][2 + c], from);
        const float v2 = __shfl_sync(0xffffffffu, o[1][c], from), v3 = __shfl_sync(0xffffffffu, o[1][2 + c], from);
        return h1 ? (hi ? v3 : v2) : (hi ? v1 : v0);
    };
    lg = fetch(os, 0, src);
    lr = fetch(oc, 0, src); lgr = fetch(oc, 1, src); lb = fetch(oc, 0, src + 1);
}

// ---- surface normals (NORMAL kernels): n = -grad(raw) / |grad(raw)| of the density logit raw = w_out . ReLU(W1 f(x))
// Data gradient of the density net for the tile, g = W1^T (m . w_out) with m = [W1 f > 0] (the fp32 layer-1 accumulator;
// the fp16 roundings of the forward count as identity): per M = 64 half one m64n32 wgmma, A = the masked output row in
// registers (the relu_frag layout of the layer-1 fragment), B = the staged W1 image read MN-major (mlp_bwd.cu).  The fp32
// result is staged into the feature tiles, idle since the last layer-1 wgmma: column chunk c (4 floats) of tile row r
// goes where k-group c % 4 of row r of feature tile c / 4 lives, so a warp writes and reads only the slots of its own
// rows (eval_row) -- no block barrier, and the next tile's encode overwrites nothing another warp still reads.
__device__ __forceinline__ uint32_t g_slot(int row, int c) { return (uint32_t)((c >> 2) * A32_BYTES + (c & 3) * A_LBO + row * 16); }

// Called after eval_mlp_regs, by all 128 threads.  The mask is the density layer 1 once more (the forward's wgmma on the
// unchanged feature tile: the same fp32 accumulator), so that no register stays live across the forward for it.
__device__ __forceinline__ void eval_density_g(const RenderSmem& sm, int tid)
{
    const int warp = tid >> 5, lane = tid & 31, q = lane & 3;
    uint32_t gm[2];                                          // bit i of gm[h]: [dg[i] > 0] of half h's fragment
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        float dg[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) dg[i] = 0.f;
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < 2; ++ks)
            wgmma_n64<0, 0>(dg, gmma_desc(smem_u32(sm.sAg) + h * 64 * 16 + ks * 2 * A_LBO, A_LBO, X_SBO),
                            gmma_desc(smem_u32(sm.sW1g) + ks * 2 * W_LBO, W_LBO, X_SBO), ks > 0 ? 1u : 0u);
        wgmma_commit();
        wgmma_wait();
        uint32_t m = 0;
#pragma unroll
        for (int i = 0; i < 32; ++i) m |= (dg[i] > 0.f ? 1u : 0u) << i;
        gm[h] = m;
    }
    wg_sync();                                               // no warp reads the feature tiles any more: g may overwrite them
    uint32_t wo[8];                                          // w_out columns 8j + 2q, +1 (fp16 pair; output image row 0)
#pragma unroll
    for (int j = 0; j < 8; ++j) wo[j] = *reinterpret_cast<const uint32_t*>(sm.sWog + j * 128 + q * 4);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        uint32_t am[16];                                     // register i = accumulator pair (2i, 2i + 1): w_out pair i / 2
#pragma unroll
        for (int i = 0; i < 16; ++i)
            am[i] = wo[i >> 1] & (((gm[h] >> (2 * i)) & 1u ? 0x0000FFFFu : 0u) | ((gm[h] >> (2 * i + 1)) & 1u ? 0xFFFF0000u : 0u));
        float d[16];
#pragma unroll
        for (int i = 0; i < 16; ++i) d[i] = 0.f;
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < 4; ++ks)                       // K = the 64 hidden units; N = the 32 features
            wgmma_n32_ra_tb(d, am + 4 * ks, gmma_desc(smem_u32(sm.sW1g) + ks * 256, 128, W_LBO), ks > 0 ? 1u : 0u);
        wgmma_commit();
        wgmma_wait();
        // d[4j + e]: row 64h + 16 warp + lane / 4 + 8 (e / 2), columns 8j + 2q + (e % 2) = chunk 2j + q / 2, float (2q) % 4 + e % 2
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
            for (int e = 0; e < 4; e += 2) {
                const int row = 64 * h + 16 * warp + (lane >> 2) + 4 * e;
                *reinterpret_cast<float2*>(sm.sA + g_slot(row, 2 * j + (q >> 1)) + (q & 1) * 8) = make_float2(d[4 * j + e], d[4 * j + e + 1]);
            }
    }
    __syncwarp();
}

// One level of d raw / d x01 (grid_grad.cuh::level_input_grad, Linear on the fast paths): the corners are addressed as the
// forward addresses them and only the geo half of each packed entry is used.  KIND as encode_group.
template <int KIND>
__device__ __forceinline__ void normal_level(const RenderArgs& a, int l, float x, float y, float z, float2 gl, float (&acc)[3])
{
    LevelFrame f;
    float2 v[8];
    if constexpr (KIND == 0) {
        level_frame(a.lt, l, x, y, z, f);
#pragma unroll
        for (int k = 0; k < 8; ++k) v[k] = unpack_half2(__ldg(&a.table[f.idx[k]].x));
    } else {
        // cell_frame's fract, kept inline: calling it changes the NORMAL kernels' SASS
        const float scale = a.lt.scale[l];
        const float in[3] = {x, y, z};
#pragma unroll
        for (int d = 0; d < 3; ++d) {
            const float pos = fmaf(scale, in[d], 0.5f);
            f.s[d] = pos - floorf(pos); f.ds[d] = 1.f; f.dds[d] = 0.f;
        }
        f.scale = scale;
        float w[8];
        if constexpr (KIND == 1) {
            const uint4* const cp = a.cells[l] + 4ull * level_cell_dense(a.lt, l, x, y, z, w);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const uint4 c2 = ldg_cell<PERF_L1_DENSE>(cp + j);
                v[2 * j] = unpack_half2(c2.x); v[2 * j + 1] = unpack_half2(c2.z);
            }
        } else {
            uint32_t idx[8];
            level_corners_rel<true>(a.lt, l, x, y, z, idx, w);
            const uint2* const tl = a.table + a.lt.offset[l];
#pragma unroll
            for (int k = 0; k < 8; ++k) v[k] = unpack_half2(__ldg(&entry_ptr(tl, idx[k])->x));
        }
    }
    level_input_grad(f, v, gl, acc);
}

// This thread's sample normal (selector true): the 16 levels again with dL/dfeature = the staged row of g, then the world
// gradient grad_d = (d raw / d x01_d) / aabb_ext_d and n = -grad / |grad| (0 when |grad| = 0).
template <int NDENSE>
__device__ __forceinline__ void sample_normal(const RenderArgs& a, const RenderSmem& sm, float x, float y, float z, int row, float (&n)[3])
{
    float acc[3] = {0.f, 0.f, 0.f};
    const uint8_t* const g_row = sm.sA + g_slot(row, 0);
    auto gl = [&](int l) { return *reinterpret_cast<const float2*>(g_row + g_slot(0, l >> 1) + (l & 1) * 8); };
    if constexpr (NDENSE == 4) {
#pragma unroll 1
        for (int l = 0; l < 4; ++l) normal_level<1>(a, l, x, y, z, gl(l), acc);
#pragma unroll 1
        for (int l = 4; l < 16; ++l) normal_level<2>(a, l, x, y, z, gl(l), acc);
    } else {
#pragma unroll 1
        for (int l = 0; l < 16; ++l) normal_level<0>(a, l, x, y, z, gl(l), acc);
    }
    const float gx = acc[0] / a.aabb_ext[0], gy = acc[1] / a.aabb_ext[1], gz = acc[2] / a.aabb_ext[2];
    const float r = fmaxf(fabsf(gx), fmaxf(fabsf(gy), fabsf(gz))) > 0.f ? rnorm3df(gx, gy, gz) : 0.f;
    n[0] = -gx * r; n[1] = -gy * r; n[2] = -gz * r;
}

// Encode + both MLPs for the warpgroup's current 128 samples (thread t = one sample at normalised position (x,y,z)); all
// 128 threads of the warpgroup call it, and its barriers (wg_sync) wait for those 128 only.
// EVAL (eval kernels: SIMT = false, SAVE = 0, eval shared-memory layout): hidden layers in registers (eval_mlp_regs), two
// barriers.  Otherwise thread t owns row t of the tiles, every layer goes through shared memory and the output
// layers run on CUDA cores (out_dots_const); 5 barriers.
// NDENSE >= 0: specialised addressing (level_corners_fast; first NDENSE levels dense, rest hashed
// power-of-two) -- branch-free and ~1/3 smaller code; NDENSE < 0: generic addressing.
// SAVE 1 / 2: also write the fp16 features and hidden activations of the density / colour network
// to row `srow` of the training buffers (srow == ~0: masked-out thread).
// Shared-memory hazards across calls: every cross-row access (the layer MMAs and their fragment stores) sits between
// barriers; everything else a thread touches is its own row.
// NORMAL (eval layout only): also nrm[3] = the sample's surface normal (sample_normal; 0 for a masked-out sample).
template <bool SIMT, int NDENSE, int SAVE, bool EVAL, bool L0SMEM = false, bool NORMAL = false>
__device__ __forceinline__ void eval_fields(const RenderArgs& a, const RenderSmem& sm, float x, float y, float z, bool selector,
                                            int tid, float& sigma, float& cr, float& cg, float& cb, uint64_t srow = ~0ull,
                                            float* nrm = nullptr)
{
    static_assert(!EVAL || (!SIMT && SAVE == 0), "the register MLP has no SIMT twin and no saves");
    static_assert(!L0SMEM || EVAL, "level 0 in shared memory: eval layout only");
    static_assert(!NORMAL || (EVAL && !L0SMEM), "normals: eval layout without level 0 in shared memory");
    uint8_t* const sA = sm.sA; uint8_t* const sAg = sm.sAg; uint8_t* const sAa = sm.sAa; uint8_t* const sH = sm.sH;
    uint8_t* const sW1g = sm.sW1g; uint8_t* const sW1a = sm.sW1a; uint8_t* const sW2a = sm.sW2a;
    const int row = EVAL ? eval_row(tid) : tid;
    if (NDENSE >= 0 && !selector) { x = 0.5f; y = 0.5f; z = 0.5f; }   // masked sample: any in-box address will do
    if constexpr (NORMAL) sm.xyz[tid] = make_float4(x, y, z, selector ? 1.f : 0.f);   // own slot: read back after the MLP
    // ---- encode both fields: 16 levels x 8 corners, one 8-byte gather per corner
    if constexpr (NDENSE == 4) {
        // dense group unrolled; the three hashed groups share ONE copy of the code (the fully
        // unrolled body stalled on instruction fetch)
        encode_group<1, SAVE, L0SMEM>(a, sm, 0, x, y, z, row, srow);
#pragma unroll 1
        for (int q = 1; q < 4; ++q) encode_group<2, SAVE>(a, sm, q, x, y, z, row, srow);
    } else {
#pragma unroll
        for (int q = 0; q < 4; ++q) encode_group<0, SAVE>(a, sm, q, x, y, z, row, srow);
    }

    if constexpr (EVAL) {
        fence_proxy_async();                                  // the feature tiles are the operand of layer 1
        wg_sync();
        float lg, lr, lgr, lb;
        eval_mlp_regs(sm, tid & 31, lg, lr, lgr, lb);
        if constexpr (NORMAL) {
            eval_density_g(sm, tid);
            const float4 p = sm.xyz[tid];
            float n[3] = {0.f, 0.f, 0.f};
            if (p.w != 0.f) sample_normal<NDENSE>(a, sm, p.x, p.y, p.z, row, n);
            __syncwarp();                                     // g is read: the next tile's encode may overwrite the slots
            nrm[0] = n[0]; nrm[1] = n[1]; nrm[2] = n[2];
        }
        sigma = selector ? expf(finish_output(lg, 0)) : 0.f;  // ngp_nerf.py:141-150
        cr = selector ? finish_output(lr, 1) : 0.f;           // ngp_nerf.py:156-161
        cg = selector ? finish_output(lgr, 1) : 0.f;
        cb = selector ? finish_output(lb, 1) : 0.f;
        return;
    }

    // ---- layer 1 of both nets: density hidden -> H, colour hidden 1 -> A (over the feature tiles)
    if constexpr (!SIMT) fence_proxy_async();
    wg_sync();
    layer_relu<SIMT>(sH, sAg, sW1g, 32, tid);
    layer_relu<SIMT, true>(sA, sAa, sW1a, 32, tid);
    if constexpr (!SIMT) fence_proxy_async();             // A is the operand of the colour layer 2
    wg_sync();

    // density: ReLU hidden -> 64-long dot -> fp16 logit -> exp     (ngp_nerf.py:141-150)
    float2 og[1] = {make_float2(0.f, 0.f)};
#pragma unroll
    for (int c = 0; c < 2; ++c) {                          // unrolled: the constant-bank offsets must be immediates
        uint32_t hp[16];
        load_chunk_canonical(sH, tid, c, hp);
        if constexpr (SAVE == 1) { if (srow != ~0ull) store_chunk_global(a.s_h1 + srow * 8, c, hp); }
        if (c == 0) out_dots_const<1, 0, 0>(hp, og); else out_dots_const<1, 0, 1>(hp, og);
    }
    sigma = selector ? expf(finish_output(out_sum(og[0]), 0)) : 0.f;

    if constexpr (SAVE == 2) {
        if (srow != ~0ull) {
#pragma unroll 1
            for (int c = 0; c < 2; ++c) { uint32_t hp[16]; load_chunk_canonical(sA, tid, c, hp); store_chunk_global(a.s_h1 + srow * 8, c, hp); }
        }
    }
    // ---- colour layer 2, in place
    layer_relu<SIMT, true>(sA, sA, sW2a, 64, tid);
    wg_sync();
    float2 oa[3] = {make_float2(0.f, 0.f), make_float2(0.f, 0.f), make_float2(0.f, 0.f)};
#pragma unroll
    for (int c = 0; c < 2; ++c) {
        uint32_t hp[16];
        load_chunk_canonical(sA, tid, c, hp);
        if constexpr (SAVE == 2) { if (srow != ~0ull) store_chunk_global(a.s_h2 + srow * 8, c, hp); }
        if (c == 0) out_dots_const<3, HID, 0>(hp, oa); else out_dots_const<3, HID, 1>(hp, oa);
    }
    cr = selector ? finish_output(out_sum(oa[0]), 1) : 0.f;      // ngp_nerf.py:156-161
    cg = selector ? finish_output(out_sum(oa[1]), 1) : 0.f;
    cb = selector ? finish_output(out_sum(oa[2]), 1) : 0.f;
}

template <bool PANO, bool SIMT>
__global__ void __launch_bounds__(TILE, 4) render_kernel(const __grid_constant__ RenderArgs a)
{
    using L = ScanLayout;                            // one warpgroup per CTA (launch_scan)
    extern __shared__ __align__(128) uint8_t smem[];
    uint8_t* wgs; const RenderSmem sm = field_smem<L>(smem, 0, wgs);
    float* const sTails = reinterpret_cast<float*>(wgs + L::TAILS);
    float* const sCarry = reinterpret_cast<float*>(wgs + L::CARRY);
    const int tid = threadIdx.x;

    stage_weights_bulk<L>(smem);                     // W1 density | W1 colour | W2 colour operand images, one bulk copy

    const uint32_t S = a.S;
    const float step = fixed_s_step(a.near, a.far, S);
    const uint64_t n_units = (a.R + a.rays_per_unit - 1) / a.rays_per_unit;
    uint32_t tile_counter = 0;

    for (uint64_t unit = blockIdx.x; unit < n_units; unit += gridDim.x) {
        for (uint32_t t = 0; t < a.tiles_per_unit; ++t, ++tile_counter) {
            const uint32_t u = t * TILE + tid;                  // sample index inside the unit
            const uint32_t ray_in_unit = u / S;
            const uint32_t k = u - ray_in_unit * S;
            const uint32_t k0_tile = (t * TILE) % S;
            const uint64_t ray = unit * a.rays_per_unit + ray_in_unit;
            const bool valid = ray < a.R;

            // ---- ray + sample position (nerf_renderer.py:127, oracle/sampler.py)
            float ox = 0.f, oy = 0.f, oz = 0.f, dx = 1.f, dy = 0.f, dz = 0.f, jit = 0.f;
            if (valid) {
                if constexpr (PANO) {
                    const int row = a.row0 + (int)(ray / (uint64_t)a.W), col = (int)(ray % (uint64_t)a.W);
                    const float yy = linspace_val(row, a.H), xx = linspace_val(col, a.W);
                    // pano_dir + rotate (common.cuh), kept inline here and below: calling them changes the render kernels' SASS
                    const float beta = -(yy - 0.5f) * 3.14159274101257324f;
                    const float alpha = -(xx - 0.5f) * 6.28318548202514648f;
                    float sa, ca, sb, cb;
                    sincosf(alpha, &sa, &ca); sincosf(beta, &sb, &cb);
                    const float cx = ca * cb, cy = sa * cb, cz = sb;
                    dx = a.pose_r[0] * cx + a.pose_r[1] * cy + a.pose_r[2] * cz;
                    dy = a.pose_r[3] * cx + a.pose_r[4] * cy + a.pose_r[5] * cz;
                    dz = a.pose_r[6] * cx + a.pose_r[7] * cy + a.pose_r[8] * cz;
                    ox = a.pose_t[0]; oy = a.pose_t[1]; oz = a.pose_t[2];
                } else {
                    ox = a.rays_o[3 * ray]; oy = a.rays_o[3 * ray + 1]; oz = a.rays_o[3 * ray + 2];
                    dx = a.rays_d[3 * ray]; dy = a.rays_d[3 * ray + 1]; dz = a.rays_d[3 * ray + 2];
                }
                if (a.training && a.jitter) jit = a.jitter[ray];
            }
            const float ts = fixed_s_t(a.near, step, k, jit), te = fixed_s_t(a.near, step, k + 1, jit);
            const float tsum = __fadd_rn(ts, te);
            const float px = sample_midpoint(ox, dx, tsum), py = sample_midpoint(oy, dy, tsum), pz = sample_midpoint(oz, dz, tsum);
            const float x = to_unit(px, a.aabb_min[0], a.aabb_ext[0]);
            const float y = to_unit(py, a.aabb_min[1], a.aabb_ext[1]);
            const float z = to_unit(pz, a.aabb_min[2], a.aabb_ext[2]);
            const bool selector = valid && x > 0.f && x < 1.f && y > 0.f && y < 1.f && z > 0.f && z < 1.f;

            float sigma, cr, cg, cb;
            eval_fields<SIMT, -1, 0, false>(a, sm, x, y, z, selector, tid, sigma, cr, cg, cb);

            // ---- composite (nerf_renderer.py:170-183; oracle/composite.py)
            const float dt = __fsub_rn(te, ts);
            const float sd = valid ? sigma * dt : 0.f;
            float* carry_prev = sCarry + (tile_counter & 1u) * 8;
            float* carry_next = sCarry + ((tile_counter + 1u) & 1u) * 8;
            const bool has_carry = (t > 0);
            float sc[1] = {sd}, sx[1];
            ray_scan<1>(sc, sx, k, k0_tile, S, tid, sTails, has_carry ? carry_prev : nullptr, carry_next);
            const float T = expf(-sx[0]);
            const float alpha = 1.f - expf(-sd);
            const float w = T * alpha;
            const float tmid = tsum * 0.5f;
            float q[5] = {w, w * tmid, w * cr, w * cg, w * cb}, qx[5];
            ray_scan<5>(q, qx, k, k0_tile, S, tid, sTails + 32, has_carry ? carry_prev + 1 : nullptr, carry_next + 1);

            if (valid && k == S - 1) {
                const float op = q[0], one_m = 1.f - op;
                float dist = q[1], r = q[2], g = q[3], b = q[4];
                if (a.training) {                                 // nerf_renderer.py:192-194
                    float n0 = 0.f, n1 = 0.f, n2 = 0.f, n3 = 0.f;
                    if (a.bg_noise) { n0 = a.bg_noise[4 * ray]; n1 = a.bg_noise[4 * ray + 1]; n2 = a.bg_noise[4 * ray + 2]; n3 = a.bg_noise[4 * ray + 3]; }
                    dist = fmaxf(dist + (n3 * 2.f - 1.f) * one_m, 0.f);
                    r += n0 * one_m; g += n1 * one_m; b += n2 * one_m;
                } else {                                          // nerf_renderer.py:195-197
                    dist += 5.f * one_m;
                    r += 0.5f * one_m; g += 0.5f * one_m; b += 0.5f * one_m;
                }
                a.rgb[3 * ray] = r; a.rgb[3 * ray + 1] = g; a.rgb[3 * ray + 2] = b;
                a.distance[ray] = dist;
                if (a.opacity) a.opacity[ray] = op;
            }
        }
    }
}


// ------------------------------------------------------------------------------------------------
// render_march_kernel: thread = RAY, the 128 rows of an MMA tile are 128 neighbouring rays at the
// same sample index k.  For a panorama a warp is an 8x4 pixel patch and a CTA a 16x8 patch, so the
// 32 lanes of every gather instruction sit next to each other in space (few distinct cache lines
// per request at the coarse and middle levels) and a thread revisits the same cells from k to k+1
// (temporal L1 reuse).  The composite is a per-thread running sum: no shuffles, no carries.
// Transmittance uses the sequential exclusive sum, the order of the oracle's cumsum.
// NORMAL: also a.normal[ray] = sum_i w_i n_i (eval layout, seg == 1).
// A CTA is blockDim.x / 128 warpgroups (launch_field), each an independent tile loop over its own shared-memory region:
// warpgroup wg of CTA b takes work items b * nwg + wg, b * nwg + wg + gridDim.x * nwg, ...
template <bool PANO, bool SIMT, int NDENSE, int SAVE = 0, bool L0SMEM = false, bool NORMAL = false>
__global__ void __launch_bounds__(WG_MAX * TILE, 1) render_march_kernel(const __grid_constant__ RenderArgs a)
{
    using L = MarchLayout<SIMT, SAVE, L0SMEM, NORMAL>;   // L::EVAL: hidden layers in registers, eval shared-memory layout
    extern __shared__ __align__(128) uint8_t smem[];
    // wg broadcast from lane 0: the compiler then knows it is warp-uniform and keeps the region's address and the wgmma
    // descriptors built from it in uniform registers (threadIdx.x / TILE alone costs the 128-register kernels spills)
    const int wg = __shfl_sync(0xffffffffu, threadIdx.x / TILE, 0), nwg = blockDim.x / TILE;
    uint8_t* wgs; const RenderSmem sm = field_smem<L>(smem, wg, wgs);
    const int tid = NORMAL ? (int)(threadIdx.x % TILE) : (int)threadIdx.x - wg * TILE, warp = tid >> 5, lane = tid & 31;

    stage_weights_bulk<L>(smem);                     // the weight operand images, one bulk copy
    if constexpr (L0SMEM) {
        uint64_t* bar2 = reinterpret_cast<uint64_t*>(smem + L::BARL0);
        if (threadIdx.x == 0) {
            mbar_init(bar2, 1); fence_mbar_init();
            asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(smem_u32(bar2)), "r"(L::L0_BYTES) : "memory");
            asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                         :: "r"(smem_u32(smem + L::L0)), "l"(a.table), "r"(L::L0_BYTES), "r"(smem_u32(bar2)) : "memory");
        }
        __syncthreads();                                   // the barrier is initialised before anyone polls it
        mbar_wait(bar2, 0);
    }

    const uint32_t S = a.S;
    // fixed_s_step, kept inline: calling it changes this kernel's SASS
    const float step = __fdiv_rn(__fsub_rn(a.far, a.near), (float)S);
    const float rext0 = __frcp_rn(a.aabb_ext[0]), rext1 = __frcp_rn(a.aabb_ext[1]), rext2 = __frcp_rn(a.aabb_ext[2]);
    // PANO, or explicit rays that form a row-major image of width a.W (perf_render_args.image_width):
    // tiles are 16x8 pixel patches; otherwise 128 consecutive rays
    const bool patch = PANO || a.W > 0;
    const int rows = patch ? (int)(a.R / (uint64_t)a.W) : 0;
    const uint32_t tiles_x = patch ? (uint32_t)patch_cols(a.W) : 0u;
    const uint32_t seg = (PANO || patch || a.pk_offsets != nullptr || a.seg == 0) ? 1u : a.seg;
    const uint32_t rpt = TILE / seg, kps = S / seg;                 // rays per tile, samples per segment
    const uint32_t my_seg = (uint32_t)tid / rpt;
    const uint64_t n_tiles = patch ? (uint64_t)tiles_x * (uint64_t)patch_rows(rows) : (a.R + rpt - 1) / rpt;

    // Work items of this warpgroup: blockIdx.x * nwg + wg, then steps of gridDim.x * nwg (n_tiles < 2^31, launch_render).
    // The normals kernels add wg inside the loop instead of into its start, and take tid from threadIdx.x % TILE: the same
    // values, but ptxas allocates the two forms differently, and each form is the one that keeps its kernels' spills
    // within what they were with one warpgroup per CTA (the others spill in the 128-register kernels).
    constexpr uint32_t wg_in_start = NORMAL ? 0u : 1u;
    for (uint32_t w0 = blockIdx.x * nwg + wg * wg_in_start; w0 + wg * (1u - wg_in_start) < n_tiles; w0 += gridDim.x * nwg) {
        const uint32_t work = w0 + wg * (1u - wg_in_start);
        // Image-shaped work is dealt out in a scattered order: the tiles in flight at any moment (4 per SM) are spread over
        // the whole image instead of forming one band of neighbouring tiles that all pull the same table lines through the
        // same L2 slices at the same time.
        const uint64_t tile = (patch && a.tile_mul > 1u) ? ((uint64_t)work * a.tile_mul) % n_tiles : work;
        // ---- this thread's ray
        uint64_t ray; bool valid;
        float ox = 0.f, oy = 0.f, oz = 0.f, dx = 1.f, dy = 0.f, dz = 0.f, jit = 0.f;
        if constexpr (PANO) {
            int prow, pcol;                                                               // prow: row inside the window
            patch_pixel(tile, tiles_x, warp, lane, prow, pcol);
            valid = prow < rows && pcol < a.W;
            ray = (uint64_t)prow * (uint64_t)a.W + (uint64_t)pcol;
            if (valid) {
                const float yy = linspace_val(a.row0 + prow, a.H), xx = linspace_val(pcol, a.W);
                const float beta = -(yy - 0.5f) * 3.14159274101257324f;
                const float alpha = -(xx - 0.5f) * 6.28318548202514648f;
                float sa, ca, sb, cb;
                sincosf(alpha, &sa, &ca); sincosf(beta, &sb, &cb);
                const float cx = ca * cb, cy = sa * cb, cz = sb;
                dx = a.pose_r[0] * cx + a.pose_r[1] * cy + a.pose_r[2] * cz;
                dy = a.pose_r[3] * cx + a.pose_r[4] * cy + a.pose_r[5] * cz;
                dz = a.pose_r[6] * cx + a.pose_r[7] * cy + a.pose_r[8] * cz;
                ox = a.pose_t[0]; oy = a.pose_t[1]; oz = a.pose_t[2];
            }
        } else {
            if (patch) {
                int prow, pcol;
                patch_pixel(tile, tiles_x, warp, lane, prow, pcol);
                valid = prow < rows && pcol < a.W;
                ray = (uint64_t)prow * (uint64_t)a.W + (uint64_t)pcol;
            } else {
                ray = tile * rpt + (uint32_t)tid % rpt;
                valid = ray < a.R;
            }
            if (valid) {
                ox = a.rays_o[3 * ray]; oy = a.rays_o[3 * ray + 1]; oz = a.rays_o[3 * ray + 2];
                dx = a.rays_d[3 * ray]; dy = a.rays_d[3 * ray + 1]; dz = a.rays_d[3 * ray + 2];
            }
        }
        if (valid && a.training && a.jitter) jit = a.jitter[ray];

        float sum_sd = 0.f;                                   // exclusive running sum of sigma*dt
        float acc_w = 0.f, acc_d = 0.f, acc_r = 0.f, acc_g = 0.f, acc_b = 0.f;
        float dl_uni = 0.f, dl_bi = 0.f;                      // distortion loss pieces (SAVE only)
        float* const acc_n = reinterpret_cast<float*>(wgs + L::NACC) + tid;  // sum w n (NORMAL only): [3][128]
        if constexpr (NORMAL) { acc_n[0] = 0.f; acc_n[TILE] = 0.f; acc_n[2 * TILE] = 0.f; }
        // packed mode: every thread walks ITS ray's samples; the tile iterates to the longest ray
        // (neighbouring rays cross the same occupied shells, so lengths inside a tile are similar)
        uint32_t n_iter = kps, my_count = S;
        int64_t pk_base = 0;
        if (!PANO && a.pk_offsets != nullptr) {
            my_count = 0;
            if (valid) { pk_base = a.pk_offsets[ray]; my_count = (uint32_t)(a.pk_offsets[ray + 1] - pk_base); }
            const uint32_t wmax = __reduce_max_sync(0xffffffffu, my_count);
            uint32_t* s_max = reinterpret_cast<uint32_t*>(wgs + L::MAX);
            wg_sync();                                        // previous tile's readers are done
            if (lane == 0) s_max[warp] = wmax;
            wg_sync();
            n_iter = max(max(s_max[0], s_max[1]), max(s_max[2], s_max[3]));
        }
#pragma unroll 1
        for (uint32_t kk = 0; kk < n_iter; ++kk) {
            const uint32_t k = my_seg * kps + kk;                 // seg == 1: k == kk
            const bool live = valid && k < my_count;
            float ts, te;
            if (!PANO && a.pk_offsets != nullptr) {
                ts = live ? a.pk_ts[pk_base + k] : 0.f; te = live ? a.pk_te[pk_base + k] : 0.f;
            } else {
                ts = fixed_s_t(a.near, step, k, jit); te = fixed_s_t(a.near, step, k + 1, jit);
            }
            const float tsum = __fadd_rn(ts, te);
            const float px = sample_midpoint(ox, dx, tsum), py = sample_midpoint(oy, dy, tsum), pz = sample_midpoint(oz, dz, tsum);
            const float x = div_uniform(__fsub_rn(px, a.aabb_min[0]), a.aabb_ext[0], rext0, a.div_generic != 0u);
            const float y = div_uniform(__fsub_rn(py, a.aabb_min[1]), a.aabb_ext[1], rext1, a.div_generic != 0u);
            const float z = div_uniform(__fsub_rn(pz, a.aabb_min[2]), a.aabb_ext[2], rext2, a.div_generic != 0u);
            const bool selector = live && x > 0.f && x < 1.f && y > 0.f && y < 1.f && z > 0.f && z < 1.f;

            float sigma, cr, cg, cb, nrm[3];
            const uint64_t srow = (SAVE != 0 && valid) ? (uint64_t)k * a.R + ray : ~0ull;
            eval_fields<SIMT, NDENSE, SAVE, L::EVAL, L0SMEM, NORMAL>(a, sm, x, y, z, selector, tid, sigma, cr, cg, cb, srow, nrm);

            const float dt = __fsub_rn(te, ts);
            const float sd = sigma * dt;
            const float T = expf(-sum_sd);
            const float w = T * (1.f - expf(-sd));
            sum_sd += sd;
            if constexpr (SAVE != 0) {
                if (valid) {
                    a.s_sigma[srow] = sigma; a.s_w[srow] = w; a.s_trans[srow] = T;
                    if constexpr (SAVE == 2) {
                        const __half2 c01 = __floats2half2_rn(cr, cg), c2 = __floats2half2_rn(cb, 0.f);
                        *reinterpret_cast<uint2*>(a.s_rgb + srow * 4) = make_uint2(*reinterpret_cast<const uint32_t*>(&c01), *reinterpret_cast<const uint32_t*>(&c2));
                    }
                }
                // torch_efficient_distloss, per ray: sum iv w^2 / 3 + 2 sum w (m W_excl - WM_excl)
                const float m = tsum * 0.5f;
                dl_uni = fmaf(dt * w, w, dl_uni);
                dl_bi = fmaf(w, m * acc_w - acc_d, dl_bi);
            }
            acc_w += w; acc_d = fmaf(w, tsum * 0.5f, acc_d);
            acc_r = fmaf(w, cr, acc_r); acc_g = fmaf(w, cg, acc_g); acc_b = fmaf(w, cb, acc_b);
            if constexpr (NORMAL) {
                float3 an = make_float3(acc_n[0], acc_n[TILE], acc_n[2 * TILE]);
                an.x = fmaf(w, nrm[0], an.x); an.y = fmaf(w, nrm[1], an.y); an.z = fmaf(w, nrm[2], an.z);
                acc_n[0] = an.x; acc_n[TILE] = an.y; acc_n[2 * TILE] = an.z;
            }
            if constexpr (SIMT) wg_sync();
        }

        bool writer = valid;
        if (seg > 1) {
            // combine the `seg` partial composites of every ray (each computed as if T = 1 at the segment
            // start): w = Toff w', Wx = Wpre + Toff Wx', ... ; scratch = the (now idle) feature tiles
            float* part = reinterpret_cast<float*>(sm.sA);
            wg_sync();
            part[0 * TILE + tid] = sum_sd; part[1 * TILE + tid] = acc_w; part[2 * TILE + tid] = acc_d;
            part[3 * TILE + tid] = acc_r;  part[4 * TILE + tid] = acc_g; part[5 * TILE + tid] = acc_b;
            part[6 * TILE + tid] = dl_uni; part[7 * TILE + tid] = dl_bi;
            wg_sync();
            writer = valid && my_seg == 0;
            if (writer) {
                float cum_sd = 0.f, W = 0.f, D = 0.f, cr = 0.f, cg = 0.f, cb = 0.f, du = 0.f, db = 0.f;
                for (uint32_t sgi = 0; sgi < seg; ++sgi) {
                    const int t = (int)(sgi * rpt) + tid;         // thread that handled segment sgi of my ray
                    const float toff = expf(-cum_sd);
                    if (SAVE != 0) a.s_toff[(uint64_t)sgi * a.R + ray] = toff;
                    const float pW = part[1 * TILE + t], pD = part[2 * TILE + t];
                    du = fmaf(toff * toff, part[6 * TILE + t], du);
                    db += toff * (W * pD - D * pW) + toff * toff * part[7 * TILE + t];
                    W = fmaf(toff, pW, W); D = fmaf(toff, pD, D);
                    cr = fmaf(toff, part[3 * TILE + t], cr); cg = fmaf(toff, part[4 * TILE + t], cg); cb = fmaf(toff, part[5 * TILE + t], cb);
                    cum_sd += part[0 * TILE + t];
                }
                acc_w = W; acc_d = D; acc_r = cr; acc_g = cg; acc_b = cb; dl_uni = du; dl_bi = db;
            }
            wg_sync();                                            // scratch is rewritten by the next tile's features
        }
        if (writer) {
            const float one_m = 1.f - acc_w;
            float dist = acc_d, r = acc_r, g = acc_g, b = acc_b;
            if constexpr (SAVE != 0) { a.s_dacc[ray] = acc_d; a.s_dl[ray] = dl_uni * (1.f / 3.f) + 2.f * dl_bi; }
            // the same background as render_kernel's; a shared helper changes this kernel's SASS
            if (a.training) {                                     // nerf_renderer.py:192-194
                float n0 = 0.f, n1 = 0.f, n2 = 0.f, n3 = 0.f;
                if (a.bg_noise) { n0 = a.bg_noise[4 * ray]; n1 = a.bg_noise[4 * ray + 1]; n2 = a.bg_noise[4 * ray + 2]; n3 = a.bg_noise[4 * ray + 3]; }
                dist = fmaxf(dist + (n3 * 2.f - 1.f) * one_m, 0.f);
                r += n0 * one_m; g += n1 * one_m; b += n2 * one_m;
            } else {                                              // nerf_renderer.py:195-197
                dist += 5.f * one_m;
                r += 0.5f * one_m; g += 0.5f * one_m; b += 0.5f * one_m;
            }
            a.rgb[3 * ray] = r; a.rgb[3 * ray + 1] = g; a.rgb[3 * ray + 2] = b;
            a.distance[ray] = dist;
            if (a.opacity) a.opacity[ray] = acc_w;
            if constexpr (NORMAL) { a.normal[3 * ray] = acc_n[0]; a.normal[3 * ray + 1] = acc_n[TILE]; a.normal[3 * ray + 2] = acc_n[2 * TILE]; }
        }
    }
}

// ------------------------------------------------------------------------------------------------
// packed_fields_kernel: both fields at PACKED samples (the output of the occupancy sampler), thread = sample,
// a tile = 128 CONSECUTIVE packed samples.  Consecutive samples of a ray are 5e-4 apart (nerf_renderer.py:151):
// a warp's 32 lanes sit in one cell of every level up to resolution ~1000, the best gather locality there is.
// Used by the fused occupancy-sampler training step (perf_train_forward_packed): writes sigma, the fp16 colour and
// the normalised position of every sample and saves the trained network's features / hidden activations at row n.
struct PackedFieldArgs {
    const int64_t* ray_indices;   // [N]
    const float*   ts;            // [N]
    const float*   te;            // [N]
    uint64_t       N;
    const int64_t* n_dev;         // optional live sample count in device memory (<= N = capacity)
    float*         sigma;         // [N]
    __half*        rgb;           // [N,4] fp16
    float*         x01;           // [N,3]
    float*         normal;        // [N,3] sample normals (NORMAL kernels)
};

// A CTA is blockDim.x / 128 warpgroups with one tile loop each, as in render_march_kernel.
template <int NDENSE, int SAVE, bool NORMAL = false>
__global__ void __launch_bounds__(WG_MAX * TILE, 1) packed_fields_kernel(const __grid_constant__ RenderArgs a, const PackedFieldArgs p)
{
    using L = MarchLayout<false, SAVE, false, NORMAL>;   // L::EVAL: hidden layers in registers, eval shared-memory layout
    extern __shared__ __align__(128) uint8_t smem[];
    const int wg = __shfl_sync(0xffffffffu, threadIdx.x / TILE, 0), nwg = blockDim.x / TILE;   // warp-uniform: see render_march_kernel
    uint8_t* wgs; const RenderSmem sm = field_smem<L>(smem, wg, wgs);
    const int tid = threadIdx.x % TILE;
    stage_weights_bulk<L>(smem);                     // the weight operand images, one bulk copy
    uint64_t N = p.N;
    if (p.n_dev) { const int64_t nd = *p.n_dev; N = nd < 0 ? 0 : ((uint64_t)nd < N ? (uint64_t)nd : N); }      // graph-replayable count
    const uint64_t n_tiles = (N + TILE - 1) / TILE;
    const float rext0 = __frcp_rn(a.aabb_ext[0]), rext1 = __frcp_rn(a.aabb_ext[1]), rext2 = __frcp_rn(a.aabb_ext[2]);
    for (uint64_t tile = (uint64_t)blockIdx.x * nwg + wg; tile < n_tiles; tile += (uint64_t)gridDim.x * nwg) {
        const uint64_t n = tile * TILE + tid;
        const bool valid = n < N;
        float x = 0.5f, y = 0.5f, z = 0.5f;
        if (valid) {
            const int64_t ray = p.ray_indices[n];
            const float tsum = __fadd_rn(p.ts[n], p.te[n]);
            const float px = sample_midpoint(a.rays_o[3 * ray], a.rays_d[3 * ray], tsum);
            const float py = sample_midpoint(a.rays_o[3 * ray + 1], a.rays_d[3 * ray + 1], tsum);
            const float pz = sample_midpoint(a.rays_o[3 * ray + 2], a.rays_d[3 * ray + 2], tsum);
            x = div_uniform(__fsub_rn(px, a.aabb_min[0]), a.aabb_ext[0], rext0, a.div_generic != 0u);
            y = div_uniform(__fsub_rn(py, a.aabb_min[1]), a.aabb_ext[1], rext1, a.div_generic != 0u);
            z = div_uniform(__fsub_rn(pz, a.aabb_min[2]), a.aabb_ext[2], rext2, a.div_generic != 0u);
        }
        const bool selector = valid && x > 0.f && x < 1.f && y > 0.f && y < 1.f && z > 0.f && z < 1.f;
        float sigma, cr, cg, cb, nrm[3];
        eval_fields<false, NDENSE, SAVE, L::EVAL, false, NORMAL>(a, sm, x, y, z, selector, tid, sigma, cr, cg, cb, valid ? n : ~0ull, nrm);
        if (valid) {
            p.sigma[n] = sigma;
            if constexpr (NORMAL) { p.normal[3 * n] = nrm[0]; p.normal[3 * n + 1] = nrm[1]; p.normal[3 * n + 2] = nrm[2]; }
            const __half2 c01 = __floats2half2_rn(cr, cg), c2 = __floats2half2_rn(cb, 0.f);
            *reinterpret_cast<uint2*>(p.rgb + n * 4) = make_uint2(*reinterpret_cast<const uint32_t*>(&c01), *reinterpret_cast<const uint32_t*>(&c2));
            // masked-out samples: the in-box stand-in position the features were taken at (their gradient is zero)
            p.x01[3 * n] = selector ? x : 0.5f; p.x01[3 * n + 1] = selector ? y : 0.5f; p.x01[3 * n + 2] = selector ? z : 0.5f;
        }
    }
}

// ------------------------------------------------------------------------------------------------
// probe_fields_kernel: both fields at positions no ray produces, the eval_fields body of packed_fields_kernel phase 0.
// LATTICE (perf_fields_lattice): the nodes of an rx x ry x rz lattice spanning the box, x01_d = i_d / (r_d - 1) exactly
// (no world round trip), sigma only.  A tile is a BRICK of 4 x 4 x 8 nodes (warp w = x plane w of the brick, its lanes
// 4 y rows x 8 z nodes, z fastest), so the corners a warp gathers at a fine level come from a few neighbouring cells,
// not from one long run along z.  Otherwise (perf_fields_points): N world points, normalised with div_uniform as the packed kernel
// does; sigma, fp16 colour and (NORMAL) the sample normal.
struct ProbeArgs {
    const float* x;               // [N,3] world points (points)
    uint64_t     N;               // points, or the slab's x planes nx (LATTICE)
    int          r[3];            // lattice resolution (LATTICE)
    int          x0;              // first x plane of the slab (LATTICE)
    uint32_t     bx, by, bz;      // bricks per axis of the slab (LATTICE)
    float*       sigma;           // [N] (points) or the slab [nx, ry, rz] (LATTICE)
    __half*      rgb;             // [N,4] fp16 (points)
    float*       normal;          // [N,3] (NORMAL)
};
constexpr int BRICK_X = 4, BRICK_Y = 4, BRICK_Z = 8;
static_assert(BRICK_X * BRICK_Y * BRICK_Z == TILE && BRICK_Y * BRICK_Z == 32, "a brick is one tile, one x plane per warp");

// A CTA is blockDim.x / 128 warpgroups with one tile loop each, as in render_march_kernel.
template <int NDENSE, bool NORMAL, bool LATTICE>
__global__ void __launch_bounds__(WG_MAX * TILE, 1) probe_fields_kernel(const __grid_constant__ RenderArgs a, const ProbeArgs p)
{
    static_assert(!(NORMAL && LATTICE), "the lattice kernel writes sigma only");
    using L = MarchLayout<false, 0, false, NORMAL>;
    extern __shared__ __align__(128) uint8_t smem[];
    const int wg = __shfl_sync(0xffffffffu, threadIdx.x / TILE, 0), nwg = blockDim.x / TILE;   // warp-uniform: see render_march_kernel
    uint8_t* wgs; const RenderSmem sm = field_smem<L>(smem, wg, wgs);
    const int tid = threadIdx.x % TILE;
    stage_weights_bulk<L>(smem);                     // the weight operand images, one bulk copy
    const uint64_t n_tiles = LATTICE ? (uint64_t)p.bx * p.by * p.bz : (p.N + TILE - 1) / TILE;
    const float rext0 = __frcp_rn(a.aabb_ext[0]), rext1 = __frcp_rn(a.aabb_ext[1]), rext2 = __frcp_rn(a.aabb_ext[2]);
    for (uint64_t tile = (uint64_t)blockIdx.x * nwg + wg; tile < n_tiles; tile += (uint64_t)gridDim.x * nwg) {
        bool valid;
        uint64_t n;                                   // output row
        float x = 0.5f, y = 0.5f, z = 0.5f;
        if constexpr (LATTICE) {
            const uint32_t bzi = (uint32_t)(tile % p.bz), byi = (uint32_t)((tile / p.bz) % p.by), bxi = (uint32_t)(tile / ((uint64_t)p.bz * p.by));
            const int li = (int)(bxi * BRICK_X) + (tid >> 5);                       // plane inside the slab
            const int j = (int)(byi * BRICK_Y) + ((tid >> 3) & 3), k = (int)(bzi * BRICK_Z) + (tid & 7);
            const int i = p.x0 + li;
            valid = li < (int)p.N && j < p.r[1] && k < p.r[2];
            n = ((uint64_t)li * p.r[1] + j) * p.r[2] + k;
            if (valid) {
                x = __fdiv_rn((float)i, (float)(p.r[0] - 1));
                y = __fdiv_rn((float)j, (float)(p.r[1] - 1));
                z = __fdiv_rn((float)k, (float)(p.r[2] - 1));
            }
        } else {
            n = tile * TILE + tid;
            valid = n < p.N;
            if (valid) {
                x = div_uniform(__fsub_rn(p.x[3 * n], a.aabb_min[0]), a.aabb_ext[0], rext0, a.div_generic != 0u);
                y = div_uniform(__fsub_rn(p.x[3 * n + 1], a.aabb_min[1]), a.aabb_ext[1], rext1, a.div_generic != 0u);
                z = div_uniform(__fsub_rn(p.x[3 * n + 2], a.aabb_min[2]), a.aabb_ext[2], rext2, a.div_generic != 0u);
            }
        }
        const bool selector = valid && x > 0.f && x < 1.f && y > 0.f && y < 1.f && z > 0.f && z < 1.f;
        float sigma, cr, cg, cb, nrm[3];
        eval_fields<false, NDENSE, 0, L::EVAL, false, NORMAL>(a, sm, x, y, z, selector, tid, sigma, cr, cg, cb, ~0ull, nrm);
        if (valid) {
            p.sigma[n] = sigma;
            if constexpr (!LATTICE) {
                if constexpr (NORMAL) { p.normal[3 * n] = nrm[0]; p.normal[3 * n + 1] = nrm[1]; p.normal[3 * n + 2] = nrm[2]; }
                const __half2 c01 = __floats2half2_rn(cr, cg), c2 = __floats2half2_rn(cb, 0.f);
                *reinterpret_cast<uint2*>(p.rgb + n * 4) = make_uint2(*reinterpret_cast<const uint32_t*>(&c01), *reinterpret_cast<const uint32_t*>(&c2));
            }
        }
    }
}

static int prepare_weights(const RenderArgs& a, cudaStream_t stream)
{
    static thread_local int sym_dev = -1; static thread_local float* sym = nullptr;
    int dev_ = 0; PERF_CUDA(cudaGetDevice(&dev_));
    if (sym_dev != dev_) { PERF_CUDA(cudaGetSymbolAddress((void**)&sym, c_wout)); sym_dev = dev_; }
    weights_prepare_kernel<<<1, 1024, 0, stream>>>(a.geo_w, a.app_w, sym);
    PERF_LAUNCH_CHECK();
    return PERF_OK;
}

static uint32_t gcd_u32(uint32_t a, uint32_t b) { while (b) { uint32_t t = a % b; a = b; b = t; } return a; }

// Dynamic shared memory of a field kernel and its shared-memory carveout: the smallest that holds `ctas` resident CTAs (the
// driver rounds the percentage up to the next size the SM supports), so that the rest of the SM's unified L1 / shared
// memory stays L1 for the table gathers.  Not left to the driver's default: the eval layout (4 warpgroups, 84.6 KB) fits the
// 100 KB carveout, which leaves 156 KB of L1 where the 228 KB one leaves 28 KB.
template <typename K>
static int set_smem(K k, int bytes, int ctas)
{
    int dev = 0, max_smem = 0, reserved = 0;
    PERF_CUDA(cudaGetDevice(&dev));
    PERF_CUDA(cudaDeviceGetAttribute(&max_smem, cudaDevAttrMaxSharedMemoryPerMultiprocessor, dev));
    PERF_CUDA(cudaDeviceGetAttribute(&reserved, cudaDevAttrReservedSharedMemoryPerBlock, dev));
    const long long need = (long long)ctas * (bytes + reserved);
    const long long pct_up = (100 * need + max_smem - 1) / max_smem;
    const int pct = pct_up < 100 ? (int)pct_up : 100;
    PERF_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
    PERF_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributePreferredSharedMemoryCarveout, pct));
    return PERF_OK;
}

// Launch of field kernel K, whose shared memory is layout L, over n_work 128-row tiles, WG_MAX tiles in flight per SM.
// nwg_max = WG_MAX (render_march_kernel, packed_fields_kernel): one CTA per SM of nwg = clamp(ceil(n_work / SMs), 1, WG_MAX)
// warpgroups that share one copy of the weights, so a small launch still spreads one tile per SM.  nwg_max = 1 (the legacy
// scan kernel): WG_MAX 128-thread CTAs per SM.  Once per device and kernel: the carveout for the nwg_max shape (set_smem),
// and a check that it is resident.  Called by launch_march, launch_packed and launch_scan only, which pick K and L together.
template <auto K, class L, class... P>
static int launch_field(int nwg_max, uint64_t n_work, cudaStream_t stream, const P&... p)
{
    static thread_local int attr_dev = -1;
    const int ctas_per_sm = WG_MAX / nwg_max;
    int dev = 0; PERF_CUDA(cudaGetDevice(&dev));
    if (attr_dev != dev) {
        const int rc = set_smem(K, L::bytes(nwg_max), ctas_per_sm); if (rc) return rc;
        int resident = 0;
        PERF_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&resident, K, nwg_max * TILE, L::bytes(nwg_max)));
        PERF_CHECK_SUP(resident >= ctas_per_sm, "field kernel: %d CTAs of %d threads and %d B of shared memory per SM, %d resident",
                       ctas_per_sm, nwg_max * TILE, L::bytes(nwg_max), resident);
        attr_dev = dev;
    }
    const uint64_t ctas = (uint64_t)num_sms() * ctas_per_sm;
    const uint64_t want = (n_work + ctas - 1) / ctas;
    const int nwg = want < (uint64_t)nwg_max ? (int)want : nwg_max;
    const uint64_t need = (n_work + nwg - 1) / nwg;
    const unsigned grid = (unsigned)(need < ctas ? need : ctas);
    K<<<grid, nwg * TILE, L::bytes(nwg), stream>>>(p...);
    return PERF_OK;
}

template <bool PANO, bool SIMT, int NDENSE, int SAVE = 0, bool L0SMEM = false, bool NORMAL = false>
static int launch_march(uint64_t n_work, cudaStream_t stream, const RenderArgs& a)
{
    return launch_field<render_march_kernel<PANO, SIMT, NDENSE, SAVE, L0SMEM, NORMAL>, MarchLayout<SIMT, SAVE, L0SMEM, NORMAL>>(WG_MAX, n_work, stream, a);
}

template <bool PANO, bool SIMT>
static int launch_scan(uint64_t n_work, cudaStream_t stream, const RenderArgs& a)
{
    return launch_field<render_kernel<PANO, SIMT>, ScanLayout>(1, n_work, stream, a);
}

template <int NDENSE, int SAVE, bool NORMAL = false>
static int launch_packed(uint64_t n_work, cudaStream_t stream, const RenderArgs& a, const PackedFieldArgs& p)
{
    return launch_field<packed_fields_kernel<NDENSE, SAVE, NORMAL>, MarchLayout<false, SAVE, false, NORMAL>>(WG_MAX, n_work, stream, a, p);
}

template <int NDENSE, bool NORMAL, bool LATTICE>
static int launch_probe(uint64_t n_work, cudaStream_t stream, const RenderArgs& a, const ProbeArgs& p)
{
    return launch_field<probe_fields_kernel<NDENSE, NORMAL, LATTICE>, MarchLayout<false, 0, false, NORMAL>>(WG_MAX, n_work, stream, a, p);
}

// The part of RenderArgs every field kernel needs: level table, packed table and its cell-major copies, weights, aabb and
// div_uniform()'s mode.  fast: PeRF's grid (4 dense + 12 hashed levels, all dense levels copied cell-major) and the caller
// did not ask for generic addressing.
static int init_field_args(const perf_render_args* args, RenderArgs& a, bool& fast)
{
    PERF_CHECK_ARG(args->d_packed_table && args->d_geo_mlp_half && args->d_app_mlp_half, "NULL table / weights");
    PERF_CHECK_ARG((uintptr_t)args->d_packed_table % 16 == 0, "misaligned table");
    uint64_t n_entries = 0;
    const int rc = build_level_table(&args->grid, &a.lt, &n_entries); if (rc) return rc;
    PERF_CHECK_SUP(args->grid.n_levels == 16, "fused field kernels need n_levels == 16 (got %u)", args->grid.n_levels);
    a.table = (const uint2*)args->d_packed_table;
    const PackedLayout pl = packed_layout(a.lt, n_entries);
    for (uint32_t l = 0; l < pl.n_cell_levels; ++l) a.cells[l] = reinterpret_cast<const uint4*>(a.table + pl.cell_start[l]);
    a.geo_w = (const __half*)args->d_geo_mlp_half; a.app_w = (const __half*)args->d_app_mlp_half;
    for (int i = 0; i < 3; ++i) { a.aabb_min[i] = args->aabb[i]; a.aabb_ext[i] = args->aabb[3 + i] - args->aabb[i]; }
    // div_uniform()'s precondition: no box extent with an all-ones significand (Markstein's exception) or out of the normal range
    a.div_generic = 0u;
    for (int i = 0; i < 3; ++i) if (!div_uniform_ok(a.aabb_ext[i])) a.div_generic = 1u;
    fast = fast_addressing_ok(a.lt, 4) && pl.n_cell_levels == 4 && (args->flags & PERF_FLAG_GENERIC_ADDR) == 0;
    return PERF_OK;
}

// The render kernel for PANO and NDENSE (4: fast addressing, -1: generic), in launch_render's order of precedence; a
// training forward (save != 0) is neither a panorama nor SIMT nor scan (launch_render refuses those).
template <bool PANO, int NDENSE>
static int render_kernels(uint64_t n_work, cudaStream_t stream, const RenderArgs& a, int save, bool normals, bool simt, bool scan, bool l0)
{
    if (normals) return launch_march<PANO, false, NDENSE, 0, false, true>(n_work, stream, a);   // eval march kernel only (the callers refuse the rest)
    if constexpr (!PANO) {
        if (save != 0) return save == 1 ? launch_march<false, false, NDENSE, 1>(n_work, stream, a) : launch_march<false, false, NDENSE, 2>(n_work, stream, a);
    }
    if (scan) return simt ? launch_scan<PANO, true>(n_work, stream, a) : launch_scan<PANO, false>(n_work, stream, a);   // legacy scan kernel
    if (simt) return launch_march<PANO, true, -1>(n_work, stream, a);
    if constexpr (PANO && NDENSE == 4) {
        if (l0) return launch_march<true, false, 4, 0, true>(n_work, stream, a);   // experiment: level 0 in shared memory, one copy per CTA
    }
    return launch_march<PANO, false, NDENSE>(n_work, stream, a);
}

// normals: a.normal is set (it shares its slot with a.s_toff, so only this flag selects the NORMAL kernels)
static int launch_render(const perf_render_args* args, RenderArgs& a, bool pano, cudaStream_t stream, int save = 0, bool normals = false)
{
    PERF_CHECK_ARG(args->d_rgb && args->d_distance, "NULL output");
    PERF_CHECK_ARG(args->n_samples >= 1 && args->n_samples <= 4096, "n_samples=%u not in [1,4096]", args->n_samples);
    PERF_CHECK_ARG(args->far > args->near, "far <= near");
    PERF_CHECK_ARG((uintptr_t)args->d_geo_mlp_half % 16 == 0 && (uintptr_t)args->d_app_mlp_half % 16 == 0, "misaligned weights");
    bool fast = false;
    int rc = init_field_args(args, a, fast); if (rc) return rc;
    a.S = args->n_samples; a.near = args->near; a.far = args->far;
    a.training = (args->flags & PERF_FLAG_TRAINING) ? 1u : 0u;
    a.jitter = args->d_jitter; a.bg_noise = args->d_bg_noise;
    a.rgb = args->d_rgb; a.distance = args->d_distance; a.opacity = args->d_opacity;
    const uint32_t g = gcd_u32(a.S, TILE);
    a.rays_per_unit = TILE / g; a.tiles_per_unit = a.S / g;       // unit = lcm(S,128) samples
    if (a.R == 0) return PERF_OK;
    const bool simt = (args->flags & PERF_FLAG_SIMT_MLP) != 0;
    const bool scan = (args->flags & PERF_FLAG_SCAN_KERNEL) != 0;
    uint64_t n_work;
#ifndef PERF_TILE_SCATTER
#define PERF_TILE_SCATTER 1
#endif
    if (scan) n_work = (a.R + a.rays_per_unit - 1) / a.rays_per_unit;
    else if (pano || a.W > 0) n_work = (uint64_t)patch_cols(a.W) * (uint64_t)patch_rows((int)(a.R / (uint64_t)a.W));
    else {
        const uint32_t rpt = TILE / (a.seg ? a.seg : 1u);
        n_work = (a.R + rpt - 1) / rpt;
    }
    PERF_CHECK_SUP(n_work < (1ull << 31), "%llu tiles of 128 rays in one launch (at most 2^31)", (unsigned long long)n_work);
    a.tile_mul = 0;
    if (PERF_TILE_SCATTER && !scan && (pano || a.W > 0) && n_work > (uint64_t)num_sms() * WG_MAX && n_work < (1ull << 31)) {
        // golden-ratio stride, made coprime with the tile count: consecutive work items land far apart, evenly spread
        uint32_t m = (uint32_t)((double)n_work * 0.6180339887498949) | 1u;
        while (m > 1u && gcd_u32(m, (uint32_t)n_work) != 1u) m += 2u;
        a.tile_mul = m % (uint32_t)n_work;
    }
    rc = prepare_weights(a, stream); if (rc) return rc;     // constant-bank output weights + operand images (c_wout, g_wimg)
    PERF_CHECK_SUP(save == 0 || (!pano && !simt && !scan), "training forward runs on the ray-marching tensor-core kernel only");
    const bool l0 = (args->flags & PERF_FLAG_L0_SMEM) != 0;
    if (pano) rc = fast ? render_kernels<true, 4>(n_work, stream, a, save, normals, simt, scan, l0) : render_kernels<true, -1>(n_work, stream, a, save, normals, simt, scan, l0);
    else      rc = fast ? render_kernels<false, 4>(n_work, stream, a, save, normals, simt, scan, l0) : render_kernels<false, -1>(n_work, stream, a, save, normals, simt, scan, l0);
    if (rc) return rc;
    PERF_LAUNCH_CHECK();
    return PERF_OK;
}

// perf_fields_packed and perf_fields_packed_normals (d_normal != null: phase 0 only)
static int fields_packed(const perf_render_args* args, const float* d_rays_o, const float* d_rays_d, const int64_t* d_ray_indices,
                         const float* d_t_starts, const float* d_t_ends, uint64_t N, const int64_t* d_n_dev, int phase, float* d_sigma, void* d_rgb_half4,
                         float* d_x01, void* d_feat, void* d_h1, void* d_h2, float* d_normal, void* stream)
{
    PERF_CHECK_ARG(args && d_rays_o && d_rays_d && d_ray_indices && d_t_starts && d_t_ends && d_sigma && d_rgb_half4 && d_x01, "NULL pointer");
    PERF_CHECK_ARG(phase == 0 || phase == PERF_PHASE_GEO || phase == PERF_PHASE_APP, "phase must be 0, PERF_PHASE_GEO or PERF_PHASE_APP");
    PERF_CHECK_ARG(phase == 0 || (d_feat && d_h1 && (phase == PERF_PHASE_GEO || d_h2)), "NULL save buffer");
    PERF_CHECK_ARG(((uintptr_t)d_feat | (uintptr_t)d_h1 | (uintptr_t)d_h2) % 16 == 0 && (uintptr_t)d_rgb_half4 % 8 == 0, "misaligned buffer");
    RenderArgs a; memset(&a, 0, sizeof(a));
    bool fast = false;
    int rc = init_field_args(args, a, fast); if (rc) return rc;
    a.rays_o = d_rays_o; a.rays_d = d_rays_d;
    a.s_feat = (uint4*)d_feat; a.s_h1 = (uint4*)d_h1; a.s_h2 = (uint4*)d_h2;
    if (N == 0) return PERF_OK;
    PackedFieldArgs p = {d_ray_indices, d_t_starts, d_t_ends, N, d_n_dev, d_sigma, (__half*)d_rgb_half4, d_x01, d_normal};
    cudaStream_t st = (cudaStream_t)stream;
    rc = prepare_weights(a, st); if (rc) return rc;
    const uint64_t n_tiles = (N + TILE - 1) / TILE;
    if (p.normal != nullptr) rc = fast ? launch_packed<4, 0, true>(n_tiles, st, a, p) : launch_packed<-1, 0, true>(n_tiles, st, a, p);
    else if (phase == 0) rc = fast ? launch_packed<4, 0>(n_tiles, st, a, p) : launch_packed<-1, 0>(n_tiles, st, a, p);
    else if (phase == PERF_PHASE_GEO) rc = fast ? launch_packed<4, 1>(n_tiles, st, a, p) : launch_packed<-1, 1>(n_tiles, st, a, p);
    else rc = fast ? launch_packed<4, 2>(n_tiles, st, a, p) : launch_packed<-1, 2>(n_tiles, st, a, p);
    if (rc) return rc;
    PERF_LAUNCH_CHECK();
    return PERF_OK;
}

// perf_render_rays and perf_render_rays_normals (d_normal != null)
static int render_rays(const perf_render_args* args, const float* d_rays_o, const float* d_rays_d, uint64_t R, float* d_normal, void* stream)
{
    PERF_CHECK_ARG(args && d_rays_o && d_rays_d, "NULL pointer");
    RenderArgs a; memset(&a, 0, sizeof(a));
    a.rays_o = d_rays_o; a.rays_d = d_rays_d; a.R = R;
    if (args->image_width > 0 && (args->flags & PERF_FLAG_SCAN_KERNEL) == 0) {
        PERF_CHECK_ARG(R % args->image_width == 0, "image_width=%u does not divide the %llu rays", args->image_width, (unsigned long long)R);
        a.W = (int)args->image_width;
    }
    a.normal = d_normal;
    return launch_render(args, a, false, (cudaStream_t)stream, 0, d_normal != nullptr);
}

// perf_render_pano and perf_render_pano_normals (d_normal != null)
static int render_pano(const perf_render_args* args, const float* h_pose, int H, int W, int row0, int rows, float* d_normal, void* stream)
{
    PERF_CHECK_ARG(args && h_pose, "NULL pointer");
    PERF_CHECK_ARG(H > 0 && W > 0 && row0 >= 0 && rows >= 0 && row0 + rows <= H, "bad panorama window H=%d W=%d row0=%d rows=%d", H, W, row0, rows);
    RenderArgs a; memset(&a, 0, sizeof(a));
    for (int r = 0; r < 3; ++r) { for (int c = 0; c < 3; ++c) a.pose_r[3 * r + c] = h_pose[4 * r + c]; a.pose_t[r] = h_pose[4 * r + 3]; }
    a.H = H; a.W = W; a.row0 = row0; a.R = (uint64_t)rows * W;
    a.normal = d_normal;
    return launch_render(args, a, true, (cudaStream_t)stream, 0, d_normal != nullptr);
}

}  // namespace perf

using namespace perf;

extern "C" {
#pragma GCC visibility push(default)

int perf_render_rays(const perf_render_args* args, const float* d_rays_o, const float* d_rays_d, uint64_t R, void* stream)
{
    return render_rays(args, d_rays_o, d_rays_d, R, nullptr, stream);
}

int perf_render_packed(const perf_render_args* args, const float* d_rays_o, const float* d_rays_d, uint64_t R,
                       const int64_t* d_offsets, const float* d_t_starts, const float* d_t_ends, void* stream)
{
    PERF_CHECK_ARG(args && d_rays_o && d_rays_d && d_offsets, "NULL pointer");
    PERF_CHECK_SUP((args->flags & (PERF_FLAG_SCAN_KERNEL | PERF_FLAG_TRAINING)) == 0, "packed rendering: eval mode on the ray-marching kernel only");
    RenderArgs a; memset(&a, 0, sizeof(a));
    a.rays_o = d_rays_o; a.rays_d = d_rays_d; a.R = R;
    a.pk_offsets = d_offsets; a.pk_ts = d_t_starts; a.pk_te = d_t_ends;
    perf_render_args t = *args; t.n_samples = 1; if (!(t.far > t.near)) { t.near = 0.f; t.far = 1.f; }
    return launch_render(&t, a, false, (cudaStream_t)stream);
}

int perf_train_forward(const perf_render_args* args, const float* d_rays_o, const float* d_rays_d, uint64_t R, int phase,
                       const perf_train_buffers* buf, void* stream)
{
    PERF_CHECK_ARG(args && d_rays_o && d_rays_d && buf, "NULL pointer");
    PERF_CHECK_ARG(phase == PERF_PHASE_GEO || phase == PERF_PHASE_APP, "phase must be PERF_PHASE_GEO or PERF_PHASE_APP");
    PERF_CHECK_ARG(buf->d_sigma && buf->d_weights && buf->d_trans && buf->d_feat && buf->d_h1 && buf->d_dist_acc && buf->d_distloss, "NULL training buffer");
    PERF_CHECK_ARG(phase == PERF_PHASE_GEO || (buf->d_rgb && buf->d_h2), "colour phase needs d_rgb and d_h2");
    PERF_CHECK_ARG(((uintptr_t)buf->d_feat | (uintptr_t)buf->d_h1 | (uintptr_t)buf->d_h2) % 16 == 0 && (uintptr_t)buf->d_rgb % 8 == 0, "misaligned training buffer");
    RenderArgs a; memset(&a, 0, sizeof(a));
    a.rays_o = d_rays_o; a.rays_d = d_rays_d; a.R = R;
    a.s_sigma = buf->d_sigma; a.s_w = buf->d_weights; a.s_trans = buf->d_trans; a.s_rgb = (__half*)buf->d_rgb;
    a.s_feat = (uint4*)buf->d_feat; a.s_h1 = (uint4*)buf->d_h1; a.s_h2 = (uint4*)buf->d_h2;
    a.s_dacc = buf->d_dist_acc; a.s_dl = buf->d_distloss;
    // split rays into segments until the tiles fill the machine (4 tiles in flight per SM), if the caller gave room
    a.seg = 1; a.s_toff = buf->d_seg_trans;
    if (buf->d_seg_trans != nullptr) {
        const uint64_t slots = (uint64_t)num_sms() * 4;
        while (a.seg < PERF_MAX_SEGMENTS && args->n_samples % (a.seg * 2) == 0 && (R * a.seg + TILE - 1) / TILE < slots) a.seg *= 2;
    }
    PERF_CHECK_ARG(buf->h_segments_out != nullptr || a.seg == 1, "d_seg_trans given without h_segments_out");
    if (buf->h_segments_out) *buf->h_segments_out = a.seg;
    perf_render_args t = *args; t.flags |= PERF_FLAG_TRAINING;
    return launch_render(&t, a, false, (cudaStream_t)stream, phase);
}


int perf_fields_packed(const perf_render_args* args, const float* d_rays_o, const float* d_rays_d, const int64_t* d_ray_indices,
                       const float* d_t_starts, const float* d_t_ends, uint64_t N, const int64_t* d_n_dev, int phase, float* d_sigma, void* d_rgb_half4,
                       float* d_x01, void* d_feat, void* d_h1, void* d_h2, void* stream)
{
    return fields_packed(args, d_rays_o, d_rays_d, d_ray_indices, d_t_starts, d_t_ends, N, d_n_dev, phase, d_sigma, d_rgb_half4, d_x01,
                         d_feat, d_h1, d_h2, nullptr, stream);
}

int perf_render_pano(const perf_render_args* args, const float* h_pose, int H, int W, int row0, int rows, void* stream)
{
    return render_pano(args, h_pose, H, W, row0, rows, nullptr, stream);
}

// ---- surface normals (perfb200.h: perf_render_pano_normals and the others)
#define PERF_NORMALS_FLAGS_OK(args) PERF_CHECK_SUP(((args)->flags & (PERF_FLAG_SIMT_MLP | PERF_FLAG_SCAN_KERNEL | PERF_FLAG_L0_SMEM | \
                                                                   PERF_FLAG_TRAINING)) == 0, "normals: eval render on the ray-marching wgmma kernel only")

int perf_render_pano_normals(const perf_render_args* args, const float* h_pose, int H, int W, int row0, int rows, float* d_normal, void* stream)
{
    PERF_CHECK_ARG(args && d_normal, "NULL pointer");
    PERF_NORMALS_FLAGS_OK(args);
    return render_pano(args, h_pose, H, W, row0, rows, d_normal, stream);
}

int perf_render_rays_normals(const perf_render_args* args, const float* d_rays_o, const float* d_rays_d, uint64_t R, float* d_normal, void* stream)
{
    PERF_CHECK_ARG(args && d_normal, "NULL pointer");
    PERF_NORMALS_FLAGS_OK(args);
    return render_rays(args, d_rays_o, d_rays_d, R, d_normal, stream);
}

int perf_fields_packed_normals(const perf_render_args* args, const float* d_rays_o, const float* d_rays_d, const int64_t* d_ray_indices,
                               const float* d_t_starts, const float* d_t_ends, uint64_t N, const int64_t* d_n_dev, float* d_sigma,
                               void* d_rgb_half4, float* d_x01, float* d_normal, void* stream)
{
    PERF_CHECK_ARG(args && d_normal, "NULL pointer");
    PERF_NORMALS_FLAGS_OK(args);
    return fields_packed(args, d_rays_o, d_rays_d, d_ray_indices, d_t_starts, d_t_ends, N, d_n_dev, 0, d_sigma, d_rgb_half4, d_x01,
                         nullptr, nullptr, nullptr, d_normal, stream);
}

// ---- fields on a lattice and at points (perfb200.h: perf_fields_lattice, perf_fields_points)
int perf_fields_lattice(const perf_render_args* args, const int* h_res3, int x0, int nx, float* d_sigma, void* stream)
{
    PERF_CHECK_ARG(args && h_res3 && d_sigma, "NULL pointer");
    PERF_CHECK_ARG(h_res3[0] >= 2 && h_res3[1] >= 2 && h_res3[2] >= 2, "lattice %d x %d x %d: every axis needs >= 2 nodes", h_res3[0], h_res3[1], h_res3[2]);
    PERF_CHECK_ARG((uint64_t)h_res3[0] * (uint64_t)h_res3[1] * (uint64_t)h_res3[2] < (1ull << 31), "lattice %d x %d x %d has >= 2^31 nodes",
                   h_res3[0], h_res3[1], h_res3[2]);
    PERF_CHECK_ARG(x0 >= 0 && nx >= 0 && x0 + nx <= h_res3[0], "x slab [%d, %d + %d) not inside [0, %d)", x0, x0, nx, h_res3[0]);
    PERF_NORMALS_FLAGS_OK(args);
    RenderArgs a; memset(&a, 0, sizeof(a));
    bool fast = false;
    int rc = init_field_args(args, a, fast); if (rc) return rc;
    if (nx == 0) return PERF_OK;
    ProbeArgs p; memset(&p, 0, sizeof(p));
    p.N = (uint64_t)nx; p.x0 = x0; p.sigma = d_sigma;
    for (int d = 0; d < 3; ++d) p.r[d] = h_res3[d];
    p.bx = (uint32_t)((nx + BRICK_X - 1) / BRICK_X); p.by = (uint32_t)((h_res3[1] + BRICK_Y - 1) / BRICK_Y); p.bz = (uint32_t)((h_res3[2] + BRICK_Z - 1) / BRICK_Z);
    cudaStream_t st = (cudaStream_t)stream;
    rc = prepare_weights(a, st); if (rc) return rc;
    const uint64_t n_tiles = (uint64_t)p.bx * p.by * p.bz;
    rc = fast ? launch_probe<4, false, true>(n_tiles, st, a, p) : launch_probe<-1, false, true>(n_tiles, st, a, p);
    if (rc) return rc;
    PERF_LAUNCH_CHECK();
    return PERF_OK;
}

int perf_fields_points(const perf_render_args* args, const float* d_x, uint64_t N, float* d_sigma, void* d_rgb_half4, float* d_normal, void* stream)
{
    PERF_CHECK_ARG(args && (N == 0 || (d_x && d_sigma && d_rgb_half4)), "NULL pointer");
    PERF_CHECK_ARG((uintptr_t)d_rgb_half4 % 8 == 0, "misaligned buffer");
    PERF_NORMALS_FLAGS_OK(args);
    RenderArgs a; memset(&a, 0, sizeof(a));
    bool fast = false;
    int rc = init_field_args(args, a, fast); if (rc) return rc;
    if (N == 0) return PERF_OK;
    ProbeArgs p; memset(&p, 0, sizeof(p));
    p.x = d_x; p.N = N; p.sigma = d_sigma; p.rgb = (__half*)d_rgb_half4; p.normal = d_normal;
    cudaStream_t st = (cudaStream_t)stream;
    rc = prepare_weights(a, st); if (rc) return rc;
    const uint64_t n_tiles = (N + TILE - 1) / TILE;
    if (d_normal != nullptr) rc = fast ? launch_probe<4, true, false>(n_tiles, st, a, p) : launch_probe<-1, true, false>(n_tiles, st, a, p);
    else rc = fast ? launch_probe<4, false, false>(n_tiles, st, a, p) : launch_probe<-1, false, false>(n_tiles, st, a, p);
    if (rc) return rc;
    PERF_LAUNCH_CHECK();
    return PERF_OK;
}
#undef PERF_NORMALS_FLAGS_OK

#pragma GCC visibility pop
}  // extern "C"
