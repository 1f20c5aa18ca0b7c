// api_basic.cu -- C-ABI entry points that are not the tensor-core paths:
// error state, level table, params cast / table packing, ray generation, stand-alone hash-grid
// encode forward / backward, packed composite (nerfacc-style) kernels, fused Adam.
#include "common.cuh"
#include <stdarg.h>
#include <stdio.h>
#include <string.h>

namespace perf {

static thread_local char g_err[512] = "";
void set_error(const char* fmt, ...)
{
    va_list ap; va_start(ap, fmt); vsnprintf(g_err, sizeof(g_err), fmt, ap); va_end(ap);
}

int num_sms()
{
    int dev = 0, n = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 148;
    static int cache[64] = {0};
    if (dev >= 0 && dev < 64 && cache[dev]) return cache[dev];
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 148;
    if (dev >= 0 && dev < 64) cache[dev] = n;
    return n;
}

// tcnn GridEncodingTemplated constructor + grid_scale/grid_resolution (SURVEY.md Appendix A);
// mirrored by oracle/hashgrid.py::level_table and asserted equal in tests/test_abi.py.
int build_level_table(const perf_grid_cfg* cfg, LevelTable* out, uint64_t* n_entries)
{
    PERF_CHECK_ARG(cfg != nullptr, "grid cfg is NULL");
    PERF_CHECK_SUP(cfg->n_levels >= 1 && cfg->n_levels <= PERF_MAX_LEVELS, "n_levels=%u not in [1,%d]", cfg->n_levels, PERF_MAX_LEVELS);
    PERF_CHECK_SUP(cfg->n_features_per_level == 2, "n_features_per_level=%u (only 2 is implemented)", cfg->n_features_per_level);
    PERF_CHECK_SUP(cfg->log2_hashmap_size >= 4 && cfg->log2_hashmap_size <= 28, "log2_hashmap_size=%u out of range", cfg->log2_hashmap_size);
    PERF_CHECK_SUP(cfg->interpolation <= 1, "interpolation=%u (0 Linear, 1 Smoothstep)", cfg->interpolation);
    PERF_CHECK_ARG(cfg->base_resolution >= 1 && cfg->per_level_scale >= 1.0f, "bad base_resolution / per_level_scale");
    LevelTable lt; memset(&lt, 0, sizeof(lt));
    lt.n_levels = cfg->n_levels; lt.smoothstep = cfg->interpolation;
    // tcnn: scale = exp2f(l * log2f(s)) * base - 1 in fp32 ON THE DEVICE; libm / CUDA exp2f differ by
    // an ulp, so the product is defined here in fp64 with ONE rounding to fp32 (libm-independent;
    // mirrored by oracle/hashgrid.py::grid_scale and property-tested in tests/test_abi.py)
    const float log2s = (float)log2((double)cfg->per_level_scale);
    uint64_t offset = 0;
    for (uint32_t l = 0; l < cfg->n_levels; ++l) {
        volatile float x = (float)l * log2s;
        const float scale = (float)(exp2((double)x) * (double)cfg->base_resolution - 1.0);
        const uint32_t res = (uint32_t)ceilf(scale) + 1u;
        const uint64_t max_params = 0xFFFFFFFFull / 2;
        uint64_t dense = ((double)res * res * res > (double)max_params) ? max_params : (uint64_t)res * res * res;
        dense = (dense + 7) / 8 * 8;
        uint64_t size = dense < (1ull << cfg->log2_hashmap_size) ? dense : (1ull << cfg->log2_hashmap_size);
        uint64_t stride = 1; int dims = 0;
        while (dims < 3 && stride <= size) { stride *= res; ++dims; }
        const bool hashed = size < stride;
        PERF_CHECK_SUP(hashed || dims == 3, "level %u: dense level with fewer than 3 strided dims", l);
        lt.scale[l] = scale; lt.res[l] = res; lt.size[l] = (uint32_t)size; lt.offset[l] = (uint32_t)offset;
        if (hashed) lt.hashed_mask |= 1u << l;
        if ((size & (size - 1)) == 0) lt.pow2_mask |= 1u << l;
        offset += size;
        PERF_CHECK_SUP(offset < (1ull << 31), "grid too large");
    }
    if (out) *out = lt;
    if (n_entries) *n_entries = offset;
    return PERF_OK;
}

int check_mlp(const perf_mlp_cfg* mlp)
{
    PERF_CHECK_ARG(mlp != nullptr, "mlp cfg is NULL");
    PERF_CHECK_SUP(mlp->n_in == 32, "mlp n_in=%u (only 32 = 16 levels x 2 features is implemented)", mlp->n_in);
    PERF_CHECK_SUP(mlp->n_neurons == 64, "mlp n_neurons=%u (only 64)", mlp->n_neurons);
    PERF_CHECK_SUP(mlp->n_hidden_layers == 1 || mlp->n_hidden_layers == 2, "mlp n_hidden_layers=%u (1 or 2)", mlp->n_hidden_layers);
    PERF_CHECK_SUP(mlp->n_out >= 1 && mlp->n_out <= 16, "mlp n_out=%u (1..16)", mlp->n_out);
    PERF_CHECK_SUP(mlp->output_activation <= 1, "mlp output_activation=%u (0 None, 1 Sigmoid)", mlp->output_activation);
    return PERF_OK;
}

int mlp_param_count(const perf_mlp_cfg* mlp, uint64_t* count)
{
    int rc = check_mlp(mlp); if (rc) return rc;
    const uint64_t padded_out = (mlp->n_out + 15) / 16 * 16;
    *count = (uint64_t)mlp->n_neurons * mlp->n_in + (uint64_t)(mlp->n_hidden_layers - 1) * mlp->n_neurons * mlp->n_neurons
           + padded_out * mlp->n_neurons;
    return PERF_OK;
}

// ------------------------------------------------------------------------------------------------
// kernels
// ------------------------------------------------------------------------------------------------
__global__ void params_to_half_kernel(const float* __restrict__ p, __half* __restrict__ h, uint64_t n)
{
    uint64_t i = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) * 4;
    if (i + 3 < n) {
        float4 v = *reinterpret_cast<const float4*>(p + i);
        uint2 o; o.x = pack_half2(v.x, v.y); o.y = pack_half2(v.z, v.w);
        *reinterpret_cast<uint2*>(h + i) = o;
    } else {
        for (; i < n; ++i) h[i] = __float2half_rn(p[i]);
    }
}

struct PackCells {            // cell-major copies of the leading dense levels (common.cuh::PackedLayout)
    uint32_t n_levels;
    uint32_t res[PERF_CELL_LEVELS], size[PERF_CELL_LEVELS], offset[PERF_CELL_LEVELS], cells[PERF_CELL_LEVELS];
    uint64_t start[PERF_CELL_LEVELS];         // first packed entry of each level's cells
};
// Threads [0, n/2): two entries each (8-byte loads from both tables, one 16-byte store).  Threads behind them: one CELL each
// -- two integer divisions, then the cell's four x-neighbour pairs as 16-byte stores (64 contiguous bytes per thread).
// Runs in front of every training step's forward (the tables changed): ~64 MB of traffic.
__global__ void __launch_bounds__(256) pack_tables_kernel(const uint32_t* __restrict__ geo, const uint32_t* __restrict__ app,
                                                          uint2* __restrict__ out, uint64_t n, const PackCells pc)
{
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t < n / 2) {
        const uint2 g = reinterpret_cast<const uint2*>(geo)[t], a = reinterpret_cast<const uint2*>(app)[t];
        reinterpret_cast<uint4*>(out)[t] = make_uint4(g.x, a.x, g.y, a.y);
        return;
    }
    uint64_t c = t - n / 2;
    int l = -1;
#pragma unroll
    for (int i = 0; i < (int)PERF_CELL_LEVELS; ++i) {              // constant indices: pc stays in the constant bank
        if (l < 0 && i < (int)pc.n_levels) { if (c < pc.cells[i]) l = i; else c -= pc.cells[i]; }
    }
    if (l < 0) return;
    uint32_t res = 0, size = 0, off = 0; uint64_t start = 0;
#pragma unroll
    for (int i = 0; i < (int)PERF_CELL_LEVELS; ++i) if (i == l) { res = pc.res[i]; size = pc.size[i]; off = pc.offset[i]; start = pc.start[i]; }
    const uint32_t cell = (uint32_t)c;
    const uint32_t gz = cell / (res * res), rem = cell - gz * res * res, gy = rem / res, gx = rem - gy * res;
    uint4* dst = reinterpret_cast<uint4*>(out + start + 8ull * cell);
#pragma unroll
    for (int q = 0; q < 4; ++q) {                                  // q = ky + 2 kz; the pair = corners (kx = 0, 1)
        uint32_t e0 = gx + res * ((gy + (q & 1)) + res * (gz + (q >> 1))), e1 = e0 + 1u;
        if (e0 >= size) e0 -= size;                                // tcnn's `% size` of a dense level (e < 2 * size)
        if (e1 >= size) e1 -= size;
        dst[q] = make_uint4(geo[off + e0], app[off + e0], geo[off + e1], app[off + e1]);
    }
}

struct Pose { float r[9]; float t[3]; };

__global__ void raygen_pano_kernel(Pose pose, int H, int W, int row0, int rows, float* __restrict__ o, float* __restrict__ d)
{
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (uint64_t)rows * W) return;
    int row = row0 + (int)(i / W), col = (int)(i % W);
    float cx, cy, cz; pano_dir(row, col, H, W, cx, cy, cz);
    rotate(pose.r, cx, cy, cz, d[3 * i + 0], d[3 * i + 1], d[3 * i + 2]);
    o[3 * i + 0] = pose.t[0]; o[3 * i + 1] = pose.t[1]; o[3 * i + 2] = pose.t[2];
}

// perspective camera rays, OpenCV convention: camera_utils.py:60-80 (cam_rays_cam_space) + :237-241
__global__ void raygen_pers_kernel(Pose pose, float span_x, float span_y, int H, int W, float* __restrict__ o, float* __restrict__ d)
{
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (uint64_t)H * W) return;
    const int row = (int)(i / W), col = (int)(i % W);
    const float y = linspace(-span_y, span_y, row, H), x = linspace(-span_x, span_x, col, W);
    const float n = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)), 1.0f));
    const float cx = x / n, cy = y / n, cz = 1.0f / n;
    rotate(pose.r, cx, cy, cz, d[3 * i + 0], d[3 * i + 1], d[3 * i + 2]);
    o[3 * i + 0] = pose.t[0]; o[3 * i + 1] = pose.t[1]; o[3 * i + 2] = pose.t[2];
}

// ---- stand-alone hash-grid encode (tcnn kernel_grid): one thread per sample, all levels.
__global__ void __launch_bounds__(256)
hashgrid_fwd_kernel(LevelTable lt, const uint32_t* __restrict__ table, const float* __restrict__ x01,
                    uint64_t N, uint32_t* __restrict__ feat)
{
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    const float x = x01[3 * i], y = x01[3 * i + 1], z = x01[3 * i + 2];
    uint32_t packed[PERF_MAX_LEVELS];
#pragma unroll
    for (int l = 0; l < PERF_MAX_LEVELS; ++l) {
        if (l < (int)lt.n_levels) {
            Corner8 c; level_corners(lt, l, x, y, z, c);
            uint32_t v[8];
#pragma unroll
            for (int k = 0; k < 8; ++k) v[k] = __ldg(table + c.idx[k]);
            packed[l] = blend8_half(c.w, v);
        }
    }
    uint32_t* dst = feat + i * lt.n_levels;
    if (lt.n_levels == 16) {
#pragma unroll
        for (int j = 0; j < 4; ++j)
            reinterpret_cast<uint4*>(dst)[j] = make_uint4(packed[4 * j], packed[4 * j + 1], packed[4 * j + 2], packed[4 * j + 3]);
    } else {
#pragma unroll
        for (int l = 0; l < PERF_MAX_LEVELS; ++l) if (l < (int)lt.n_levels) dst[l] = packed[l];
    }
}

// ---- hash-grid backward (tcnn kernel_grid_backward): dtable[idx] += w * dfeat, float2 atomics.
// One thread per (sample, level): the threads of a warp work on the same level of neighbouring
// samples.  MERGE (coarse levels): samples arrive ray-major, so neighbouring lanes usually sit in the
// SAME cell (a level-0 cell holds ~17 consecutive samples of a ray); runs of equal cells are summed
// with a segmented warp scan and only the last lane of a run issues the 8 atomics -- this removes
// most of the same-address traffic on the few coarse cells every ray crosses near the camera.
template <bool MERGE>
__global__ void __launch_bounds__(256)
hashgrid_bwd_kernel(LevelTable lt, int level0, const float* __restrict__ x01, const float* __restrict__ dfeat,
                    uint64_t N, float2* __restrict__ dtable, const int64_t* __restrict__ n_dev = nullptr)
{
    if (n_dev) { const int64_t nd = *n_dev; N = nd < 0 ? 0 : ((uint64_t)nd < N ? (uint64_t)nd : N); }       // graph-replayable row count
    const int l = level0 + blockIdx.y, lane = threadIdx.x & 31;
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const bool live = i < N;
    float2 g = make_float2(0.f, 0.f);
    float x = 0.5f, y = 0.5f, z = 0.5f;
    if (live) {
        g = *reinterpret_cast<const float2*>(dfeat + i * (2 * lt.n_levels) + 2 * l);
        x = x01[3 * i]; y = x01[3 * i + 1]; z = x01[3 * i + 2];
    }
    const bool active = live && (g.x != 0.f || g.y != 0.f);
    if (!MERGE && !active) return;
    const float scale = lt.scale[l];
    const uint32_t res = lt.res[l], size = lt.size[l], off = lt.offset[l];
    const bool hashed = (lt.hashed_mask >> l) & 1u, pow2 = (lt.pow2_mask >> l) & 1u;
    const float px = fmaf(scale, x, 0.5f), py = fmaf(scale, y, 0.5f), pz = fmaf(scale, z, 0.5f);
    const float fx = floorf(px), fy = floorf(py), fz = floorf(pz);
    const uint32_t gx = (uint32_t)(int)fx, gy = (uint32_t)(int)fy, gz = (uint32_t)(int)fz;
    float wx = px - fx, wy = py - fy, wz = pz - fz;
    if (lt.smoothstep) { wx = wx * wx * (3.f - 2.f * wx); wy = wy * wy * (3.f - 2.f * wy); wz = wz * wz * (3.f - 2.f * wz); }
    const float ox = 1.f - wx, oy = 1.f - wy, oz = 1.f - wz;
    float2 v[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const float w = active ? __fmul_rn(__fmul_rn((k & 1) ? wx : ox, (k & 2) ? wy : oy), (k & 4) ? wz : oz) : 0.f;
        v[k] = make_float2(w * g.x, w * g.y);
    }
    bool tail = true;
    if constexpr (MERGE) {
        const uint32_t pgx = __shfl_up_sync(0xffffffffu, gx, 1), pgy = __shfl_up_sync(0xffffffffu, gy, 1), pgz = __shfl_up_sync(0xffffffffu, gz, 1);
        const bool pact = __shfl_up_sync(0xffffffffu, (int)active, 1) != 0;
        const bool head = lane == 0 || !active || !pact || pgx != gx || pgy != gy || pgz != gz;
        const uint32_t heads = __ballot_sync(0xffffffffu, head);
        const int seg_start = 31 - __clz(heads & (0xffffffffu >> (31 - lane)));
#pragma unroll
        for (int offs = 1; offs < 32; offs <<= 1) {
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                const float tx = __shfl_up_sync(0xffffffffu, v[k].x, offs), ty = __shfl_up_sync(0xffffffffu, v[k].y, offs);
                if (lane - offs >= seg_start) { v[k].x += tx; v[k].y += ty; }
            }
        }
        tail = lane == 31 || ((heads >> (lane + 1)) & 1u);
    }
    if (active && tail) {
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const uint32_t idx = off + level_index(gx + (k & 1), gy + ((k >> 1) & 1), gz + ((k >> 2) & 1), hashed, pow2, res, size);
            atomicAdd(dtable + idx, v[k]);
        }
    }
}

// ---- batch draw: rows idx[b] of up to 6 row-major fp32 arrays in ONE launch (sup_info.py:253-259 gathers rays_o, rays_d,
// colours, distances, normals with the same index vector: 5-6 index kernels per training step otherwise)
struct GatherArgs { const float* src[6]; float* dst[6]; int width[6]; int n_arrays; const int64_t* idx; uint64_t B;
                    const double* csum; uint64_t M; int64_t* idx_out; };
__global__ void __launch_bounds__(256) gather_rows_kernel(const GatherArgs a)
{
    const uint64_t b = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= a.B) return;
    int64_t r;
    if (a.csum) {
        // sorted uniform draw: csum = running sums S_1 .. S_{B+1} of i.i.d. Exp(1); S_k / S_{B+1}, k = 1..B, are distributed as the
        // ORDER STATISTICS of B i.i.d. U(0,1) -- the batch torch.randint + sort would give, without the sort
        r = (int64_t)(a.csum[b] / a.csum[a.B] * (double)a.M);
        r = r < 0 ? 0 : (r > (int64_t)a.M - 1 ? (int64_t)a.M - 1 : r);
        if (a.idx_out) a.idx_out[b] = r;
    } else {
        r = a.idx[b];
    }
    for (int k = 0; k < a.n_arrays; ++k) {
        const int w = a.width[k];
        const float* s = a.src[k] + (uint64_t)r * w; float* d = a.dst[k] + b * w;
        for (int j = 0; j < w; ++j) d[j] = s[j];
    }
}

// ---- diagnostics: the L2 atomic rate the grid-gradient scatter is bounded by (bench.py train_roofline denominator).
// Every thread issues `per_thread` reductions of `VEC` floats at pseudo-random VEC-aligned slots of a table (no other work).
template <int VEC>
__global__ void __launch_bounds__(256) atomic_rate_kernel(float* __restrict__ table, uint32_t n_slots, int per_thread)
{
    uint32_t x = (blockIdx.x * blockDim.x + threadIdx.x) * 2654435761u + 12345u;
    for (int i = 0; i < per_thread; ++i) {
        x ^= x << 13; x ^= x >> 17; x ^= x << 5;                       // xorshift32
        const uint32_t slot = x % n_slots;
        if constexpr (VEC == 4) atomicAdd(reinterpret_cast<float4*>(table) + slot, make_float4(1.f, 1.f, 1.f, 1.f));
        else if constexpr (VEC == 2) atomicAdd(reinterpret_cast<float2*>(table) + slot, make_float2(1.f, 1.f));
        else atomicAdd(table + slot, 1.f);
    }
}

// ---- packed composite kernels (nerfacc semantics): one warp per ray, lanes over its samples.
__device__ __forceinline__ uint64_t lower_bound_i64(const int64_t* a, uint64_t n, int64_t key)
{
    uint64_t lo = 0, hi = n;
    while (lo < hi) { uint64_t mid = (lo + hi) >> 1; if (a[mid] < key) lo = mid + 1; else hi = mid; }
    return lo;
}

__device__ __forceinline__ float warp_incl_scan(float v, int lane)
{
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) { float t = __shfl_up_sync(0xffffffffu, v, off); if (lane >= off) v += t; }
    return v;
}
__device__ __forceinline__ float warp_sum(float v)
{
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
    return v;
}

__global__ void __launch_bounds__(256)
weights_from_density_kernel(const float* __restrict__ ts, const float* __restrict__ te, const float* __restrict__ sig,
                            const int64_t* __restrict__ ri, uint64_t N, uint64_t n_rays,
                            float* __restrict__ w_out, float* __restrict__ T_out, float* __restrict__ a_out)
{
    const int lane = threadIdx.x & 31;
    const uint64_t ray = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (ray >= n_rays) return;
    const uint64_t s = lower_bound_i64(ri, N, (int64_t)ray), e = lower_bound_i64(ri, N, (int64_t)ray + 1);
    float carry = 0.f;
    for (uint64_t b = s; b < e; b += 32) {
        const uint64_t i = b + lane;
        const bool ok = i < e;
        const float sd = ok ? sig[i] * (te[i] - ts[i]) : 0.f;
        const float inc = warp_incl_scan(sd, lane);
        float exc = __shfl_up_sync(0xffffffffu, inc, 1); if (lane == 0) exc = 0.f;
        if (ok) {
            const float Tq = expf(-(carry + exc));
            const float a = 1.f - expf(-sd);
            if (w_out) w_out[i] = Tq * a;
            if (T_out) T_out[i] = Tq;
            if (a_out) a_out[i] = a;
        }
        carry += __shfl_sync(0xffffffffu, inc, 31);
    }
}

// dL/dsigma_i = dt_i * [ (T_i - w_i) gw_i - sum_{j>i} (w_j gw_j + T_j gT_j) ]      (SURVEY Appendix B)
__global__ void __launch_bounds__(256)
weights_from_density_bwd_kernel(const float* __restrict__ ts, const float* __restrict__ te,
                                const int64_t* __restrict__ ri, uint64_t N, uint64_t n_rays,
                                const float* __restrict__ w, const float* __restrict__ T,
                                const float* __restrict__ gw, const float* __restrict__ gT, float* __restrict__ gsig)
{
    const int lane = threadIdx.x & 31;
    const uint64_t ray = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (ray >= n_rays) return;
    const uint64_t s = lower_bound_i64(ri, N, (int64_t)ray), e = lower_bound_i64(ri, N, (int64_t)ray + 1);
    if (e == s) return;
    float carry = 0.f;                                   // sum over samples after the current chunk
    const uint64_t n = e - s, nchunks = (n + 31) / 32;
    for (uint64_t cidx = nchunks; cidx-- > 0;) {
        // reversed lane order inside the chunk: lane 0 holds the LAST sample of the chunk
        const uint64_t i = s + cidx * 32 + (31 - lane);
        const bool ok = i < e;
        const float wi = ok ? w[i] : 0.f, Ti = ok ? T[i] : 0.f;
        const float gwi = ok ? gw[i] : 0.f, gTi = (ok && gT) ? gT[i] : 0.f;
        const float term = wi * gwi + Ti * gTi;
        const float inc = warp_incl_scan(term, lane);
        float exc = __shfl_up_sync(0xffffffffu, inc, 1); if (lane == 0) exc = 0.f;
        if (ok) gsig[i] = (te[i] - ts[i]) * ((Ti - wi) * gwi - (carry + exc));
        carry += __shfl_sync(0xffffffffu, inc, 31);
    }
}

__global__ void __launch_bounds__(256)
accumulate_along_rays_kernel(const float* __restrict__ w, const float* __restrict__ v, int D,
                             const int64_t* __restrict__ ri, uint64_t N, uint64_t n_rays, float* __restrict__ out)
{
    const int lane = threadIdx.x & 31;
    const uint64_t ray = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (ray >= n_rays) return;
    const uint64_t s = lower_bound_i64(ri, N, (int64_t)ray), e = lower_bound_i64(ri, N, (int64_t)ray + 1);
    for (int d = 0; d < D; ++d) {
        float acc = 0.f;
        for (uint64_t i = s + lane; i < e; i += 32) acc += v ? w[i] * v[i * D + d] : w[i];
        acc = warp_sum(acc);
        if (lane == 0) out[ray * D + d] = acc;
    }
}

struct Scalars8 { float v[8]; };
__global__ void set_scalars_kernel(float* dst, Scalars8 s, int n) { if ((int)threadIdx.x < n) dst[threadIdx.x] = s.v[threadIdx.x]; }

// ---- fused Adam (torch.optim.Adam semantics, amsgrad=False, weight_decay=0) + fp16 shadow.
// `hyper` (device, optional): {lr, 1 - beta1^t, sqrt(1 - beta2^t)} read at run time, so a CUDA graph
// holding this launch can be replayed with a new learning rate / step count.
__device__ __forceinline__ float adam_one(float& p, float g, float& m, float& v, float lr_bc1, float b1, float b2, float eps, float bc2_sqrt, float gscale)
{
    const float gi = g * gscale;
    const float mi = b1 * m + (1.f - b1) * gi;          // exp_avg.lerp_(grad, 1-beta1)
    const float vi = b2 * v + (1.f - b2) * gi * gi;     // exp_avg_sq.mul_(b2).addcmul_(g, g, 1-b2)
    m = mi; v = vi;
    const float denom = sqrtf(vi) / bc2_sqrt + eps;
    p = p - lr_bc1 * (mi / denom);
    return p;
}

// Four parameters per thread (16-byte loads / stores, 8-byte shadow store): the pass is pure streaming, 30 B per
// parameter.  `n4` float4 groups + a scalar tail.
__global__ void __launch_bounds__(256)
adam_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
            __half* __restrict__ ph, uint64_t n, float lr, float b1, float b2, float eps,
            float bc1, float bc2_sqrt, float gscale, const float* __restrict__ hyper, int vec)
{
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (hyper) { lr = hyper[0]; bc1 = hyper[1]; bc2_sqrt = hyper[2]; }
    const float lr_bc1 = lr / bc1;
    const uint64_t n4 = vec ? n / 4 : 0;
    if (t < n4) {
        float4 pp = reinterpret_cast<float4*>(p)[t], mm = reinterpret_cast<float4*>(m)[t], vv = reinterpret_cast<float4*>(v)[t];
        const float4 gg = reinterpret_cast<const float4*>(g)[t];
        adam_one(pp.x, gg.x, mm.x, vv.x, lr_bc1, b1, b2, eps, bc2_sqrt, gscale);
        adam_one(pp.y, gg.y, mm.y, vv.y, lr_bc1, b1, b2, eps, bc2_sqrt, gscale);
        adam_one(pp.z, gg.z, mm.z, vv.z, lr_bc1, b1, b2, eps, bc2_sqrt, gscale);
        adam_one(pp.w, gg.w, mm.w, vv.w, lr_bc1, b1, b2, eps, bc2_sqrt, gscale);
        reinterpret_cast<float4*>(p)[t] = pp; reinterpret_cast<float4*>(m)[t] = mm; reinterpret_cast<float4*>(v)[t] = vv;
        if (ph) {
            const __half2 h01 = __floats2half2_rn(pp.x, pp.y), h23 = __floats2half2_rn(pp.z, pp.w);
            reinterpret_cast<uint2*>(ph)[t] = make_uint2(*reinterpret_cast<const uint32_t*>(&h01), *reinterpret_cast<const uint32_t*>(&h23));
        }
    }
    const uint64_t i = n4 * 4 + t;                       // scalar tail (or everything when the buffers are not 16-byte aligned)
    if (i < n && t < n - n4 * 4) {
        float pi = p[i], mi = m[i], vi = v[i];
        adam_one(pi, g[i], mi, vi, lr_bc1, b1, b2, eps, bc2_sqrt, gscale);
        p[i] = pi; m[i] = mi; v[i] = vi;
        if (ph) ph[i] = __float2half_rn(pi);
    }
}

// grid for adam_kernel: covers max(n/4 groups, tail elements)
static inline bool adam_vec_ok(const void* p, const void* g, const void* m, const void* v, const void* ph)
{
    return (((uintptr_t)p | (uintptr_t)g | (uintptr_t)m | (uintptr_t)v) % 16 == 0) && ((uintptr_t)ph % 8 == 0);
}

}  // namespace perf

// ------------------------------------------------------------------------------------------------
// C-ABI
// ------------------------------------------------------------------------------------------------
using namespace perf;
static inline cudaStream_t S(void* s) { return reinterpret_cast<cudaStream_t>(s); }
static inline unsigned blocks_for(uint64_t n, unsigned per) { return (unsigned)((n + per - 1) / per); }

extern "C" {
#pragma GCC visibility push(default)

int perf_abi_version(void) { return PERF_ABI_VERSION; }
const char* perf_last_error(void) { return perf::g_err; }

int perf_device_arch(void)
{
    int dev = 0, major = 0, minor = 0;
    PERF_CUDA(cudaGetDevice(&dev));
    PERF_CUDA(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev));
    PERF_CUDA(cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev));
    return major * 10 + minor;
}

int perf_grid_describe(const perf_grid_cfg* cfg, perf_level* h_levels, uint64_t* h_n_entries)
{
    LevelTable lt; uint64_t n = 0;
    int rc = build_level_table(cfg, &lt, &n); if (rc) return rc;
    if (h_levels)
        for (uint32_t l = 0; l < lt.n_levels; ++l) {
            h_levels[l].scale = lt.scale[l]; h_levels[l].resolution = lt.res[l]; h_levels[l].size = lt.size[l];
            h_levels[l].offset = lt.offset[l]; h_levels[l].hashed = (lt.hashed_mask >> l) & 1u;
        }
    if (h_n_entries) *h_n_entries = n;
    return PERF_OK;
}

int perf_network_param_count(const perf_grid_cfg* grid, const perf_mlp_cfg* mlp, uint64_t* h_count)
{
    PERF_CHECK_ARG(h_count != nullptr, "h_count is NULL");
    uint64_t ne = 0, nm = 0;
    int rc = build_level_table(grid, nullptr, &ne); if (rc) return rc;
    rc = mlp_param_count(mlp, &nm); if (rc) return rc;
    *h_count = nm + ne * grid->n_features_per_level;
    return PERF_OK;
}

int perf_params_to_half(const float* d_params, void* d_params_half, uint64_t n, void* stream)
{
    PERF_CHECK_ARG(d_params && d_params_half, "NULL pointer");
    PERF_CHECK_ARG(((uintptr_t)d_params % 16 == 0) && ((uintptr_t)d_params_half % 8 == 0), "params must be 16-byte aligned");
    if (n == 0) return PERF_OK;
    params_to_half_kernel<<<blocks_for((n + 3) / 4, 256), 256, 0, S(stream)>>>(d_params, (__half*)d_params_half, n);
    PERF_LAUNCH_CHECK();
    return PERF_OK;
}

int perf_packed_table_entries(const perf_grid_cfg* cfg, uint64_t* h_entries)
{
    PERF_CHECK_ARG(h_entries != nullptr, "NULL pointer");
    LevelTable lt; uint64_t ne = 0;
    int rc = build_level_table(cfg, &lt, &ne); if (rc) return rc;
    *h_entries = packed_layout(lt, ne).total_entries;
    return PERF_OK;
}

int perf_pack_tables(const perf_grid_cfg* grid, const perf_mlp_cfg* geo_mlp, const perf_mlp_cfg* app_mlp,
                     const void* d_geo_params_half, const void* d_app_params_half, void* d_packed, void* stream)
{
    PERF_CHECK_ARG(d_geo_params_half && d_app_params_half && d_packed, "NULL pointer");
    uint64_t ne = 0, ng = 0, na = 0;
    LevelTable lt;
    int rc = build_level_table(grid, &lt, &ne); if (rc) return rc;
    rc = mlp_param_count(geo_mlp, &ng); if (rc) return rc;
    rc = mlp_param_count(app_mlp, &na); if (rc) return rc;
    const uint32_t* geo = reinterpret_cast<const uint32_t*>((const __half*)d_geo_params_half + ng);
    const uint32_t* app = reinterpret_cast<const uint32_t*>((const __half*)d_app_params_half + na);
    PERF_CHECK_ARG(((uintptr_t)geo % 8 == 0) && ((uintptr_t)app % 8 == 0) && ((uintptr_t)d_packed % 16 == 0) && ne % 2 == 0, "misaligned tables (grids 8-byte, d_packed 16-byte aligned)");
    const PackedLayout pl = packed_layout(lt, ne);
    PackCells pc; memset(&pc, 0, sizeof(pc));
    pc.n_levels = pl.n_cell_levels;
    uint64_t n_cells = 0;
    for (uint32_t l = 0; l < pl.n_cell_levels; ++l) {
        pc.res[l] = lt.res[l]; pc.size[l] = lt.size[l]; pc.offset[l] = lt.offset[l]; pc.start[l] = pl.cell_start[l];
        pc.cells[l] = lt.res[l] * lt.res[l] * lt.res[l]; n_cells += pc.cells[l];
    }
    pack_tables_kernel<<<blocks_for(ne / 2 + n_cells, 256), 256, 0, S(stream)>>>(geo, app, (uint2*)d_packed, ne, pc);
    PERF_LAUNCH_CHECK();
    return PERF_OK;
}

int perf_raygen_pano(const float* h_pose, int H, int W, int row0, int rows, float* d_rays_o, float* d_rays_d, void* stream)
{
    PERF_CHECK_ARG(h_pose && d_rays_o && d_rays_d, "NULL pointer");
    PERF_CHECK_ARG(H > 0 && W > 0 && row0 >= 0 && rows >= 0 && row0 + rows <= H, "bad panorama window H=%d W=%d row0=%d rows=%d", H, W, row0, rows);
    if (rows == 0) return PERF_OK;
    Pose p;
    for (int r = 0; r < 3; ++r) { for (int c = 0; c < 3; ++c) p.r[3 * r + c] = h_pose[4 * r + c]; p.t[r] = h_pose[4 * r + 3]; }
    raygen_pano_kernel<<<blocks_for((uint64_t)rows * W, 256), 256, 0, S(stream)>>>(p, H, W, row0, rows, d_rays_o, d_rays_d);
    PERF_LAUNCH_CHECK();
    return PERF_OK;
}

int perf_raygen_pers(const float* h_pose, float fovy, int H, int W, float* d_rays_o, float* d_rays_d, void* stream)
{
    PERF_CHECK_ARG(h_pose && d_rays_o && d_rays_d, "NULL pointer");
    PERF_CHECK_ARG(H > 0 && W > 0 && fovy > 0.f && fovy < 3.14159f, "bad perspective camera H=%d W=%d fovy=%f", H, W, fovy);
    Pose p;
    for (int r = 0; r < 3; ++r) { for (int c = 0; c < 3; ++c) p.r[3 * r + c] = h_pose[4 * r + c]; p.t[r] = h_pose[4 * r + 3]; }
    const double span_y = tan((double)fovy * 0.5), span_x = span_y * ((double)W / (double)H);
    raygen_pers_kernel<<<blocks_for((uint64_t)H * W, 256), 256, 0, S(stream)>>>(p, (float)span_x, (float)span_y, H, W, d_rays_o, d_rays_d);
    PERF_LAUNCH_CHECK();
    return PERF_OK;
}

int perf_hashgrid_fwd(const perf_grid_cfg* cfg, const void* d_table, const float* d_x01, uint64_t N, void* d_feat, void* stream)
{
    PERF_CHECK_ARG(d_table && d_x01 && d_feat, "NULL pointer");
    LevelTable lt; int rc = build_level_table(cfg, &lt, nullptr); if (rc) return rc;
    PERF_CHECK_ARG((uintptr_t)d_table % 4 == 0 && (uintptr_t)d_feat % 16 == 0, "misaligned table/feat");
    if (N == 0) return PERF_OK;
    hashgrid_fwd_kernel<<<blocks_for(N, 256), 256, 0, S(stream)>>>(lt, (const uint32_t*)d_table, d_x01, N, (uint32_t*)d_feat);
    PERF_LAUNCH_CHECK();
    return PERF_OK;
}

int perf_hashgrid_bwd(const perf_grid_cfg* cfg, const float* d_x01, const float* d_dfeat, uint64_t N, float* d_dtable, void* stream)
{
    PERF_CHECK_ARG(d_x01 && d_dfeat && d_dtable, "NULL pointer");
    LevelTable lt; int rc = build_level_table(cfg, &lt, nullptr); if (rc) return rc;
    PERF_CHECK_ARG((uintptr_t)d_dtable % 8 == 0 && (uintptr_t)d_dfeat % 8 == 0, "misaligned dtable/dfeat");
    if (N == 0) return PERF_OK;
    // levels whose cells span several consecutive samples of a ray: merge runs; the rest: direct atomics
    const uint32_t n_merge = lt.n_levels < 6 ? lt.n_levels : 6;
    hashgrid_bwd_kernel<true><<<dim3(blocks_for(N, 256), n_merge), 256, 0, S(stream)>>>(lt, 0, d_x01, d_dfeat, N, (float2*)d_dtable);
    PERF_LAUNCH_CHECK();
    if (lt.n_levels > n_merge) {
        hashgrid_bwd_kernel<false><<<dim3(blocks_for(N, 256), lt.n_levels - n_merge), 256, 0, S(stream)>>>(lt, (int)n_merge, d_x01, d_dfeat, N, (float2*)d_dtable);
        PERF_LAUNCH_CHECK();
    }
    return PERF_OK;
}

int perf_gather_rows(const int64_t* d_idx, uint64_t B, int n_arrays, const float* const* h_src, float* const* h_dst, const int* h_width, void* stream)
{
    PERF_CHECK_ARG(d_idx && h_src && h_dst && h_width && n_arrays >= 1 && n_arrays <= 6, "bad arguments");
    GatherArgs a; memset(&a, 0, sizeof(a));
    for (int k = 0; k < n_arrays; ++k) {
        PERF_CHECK_ARG(h_src[k] && h_dst[k] && h_width[k] >= 1 && h_width[k] <= 64, "bad array %d", k);
        a.src[k] = h_src[k]; a.dst[k] = h_dst[k]; a.width[k] = h_width[k];
    }
    a.n_arrays = n_arrays; a.idx = d_idx; a.B = B;
    if (B == 0) return PERF_OK;
    gather_rows_kernel<<<blocks_for(B, 256), 256, 0, S(stream)>>>(a);
    PERF_LAUNCH_CHECK();
    return PERF_OK;
}

int perf_draw_gather_rows(const double* d_csum, uint64_t B, uint64_t M, int64_t* d_idx_out, int n_arrays, const float* const* h_src,
                          float* const* h_dst, const int* h_width, void* stream)
{
    PERF_CHECK_ARG(d_csum && h_src && h_dst && h_width && n_arrays >= 1 && n_arrays <= 6 && M >= 1, "bad arguments");
    GatherArgs a; memset(&a, 0, sizeof(a));
    for (int k = 0; k < n_arrays; ++k) {
        PERF_CHECK_ARG(h_src[k] && h_dst[k] && h_width[k] >= 1 && h_width[k] <= 64, "bad array %d", k);
        a.src[k] = h_src[k]; a.dst[k] = h_dst[k]; a.width[k] = h_width[k];
    }
    a.n_arrays = n_arrays; a.B = B; a.csum = d_csum; a.M = M; a.idx_out = d_idx_out;
    if (B == 0) return PERF_OK;
    gather_rows_kernel<<<blocks_for(B, 256), 256, 0, S(stream)>>>(a);
    PERF_LAUNCH_CHECK();
    return PERF_OK;
}

int perf_debug_atomic_rate(float* d_table, uint64_t n_floats, uint64_t n_atomics, int vec, void* stream)
{
    PERF_CHECK_ARG(d_table && (vec == 1 || vec == 2 || vec == 4) && n_floats >= 4 && (uintptr_t)d_table % 16 == 0, "bad arguments");
    const int per_thread = 16;
    const uint64_t threads = (n_atomics + per_thread - 1) / per_thread;
    const uint32_t n_slots = (uint32_t)(n_floats / vec);
    const unsigned grid = blocks_for(threads, 256);
    if (vec == 4) atomic_rate_kernel<4><<<grid, 256, 0, S(stream)>>>(d_table, n_slots, per_thread);
    else if (vec == 2) atomic_rate_kernel<2><<<grid, 256, 0, S(stream)>>>(d_table, n_slots, per_thread);
    else atomic_rate_kernel<1><<<grid, 256, 0, S(stream)>>>(d_table, n_slots, per_thread);
    PERF_LAUNCH_CHECK();
    return PERF_OK;
}

int perf_hashgrid_bwd_merged(const perf_grid_cfg* cfg, const float* d_x01, const float* d_dfeat, uint64_t N, const int64_t* d_n_dev,
                             float* d_dtable, uint32_t n_merge_levels, void* stream)
{
    PERF_CHECK_ARG(cfg && d_x01 && d_dfeat && d_dtable, "NULL pointer");
    LevelTable lt; int rc = build_level_table(cfg, &lt, nullptr); if (rc) return rc;
    PERF_CHECK_ARG((uintptr_t)d_dtable % 8 == 0 && (uintptr_t)d_dfeat % 8 == 0, "misaligned dtable/dfeat");
    if (N == 0) return PERF_OK;
    const uint32_t n_merge = n_merge_levels < lt.n_levels ? n_merge_levels : lt.n_levels;
    if (n_merge > 0) {
        hashgrid_bwd_kernel<true><<<dim3(blocks_for(N, 256), n_merge), 256, 0, S(stream)>>>(lt, 0, d_x01, d_dfeat, N, (float2*)d_dtable, d_n_dev);
        PERF_LAUNCH_CHECK();
    }
    if (lt.n_levels > n_merge) {
        hashgrid_bwd_kernel<false><<<dim3(blocks_for(N, 256), lt.n_levels - n_merge), 256, 0, S(stream)>>>(lt, (int)n_merge, d_x01, d_dfeat, N, (float2*)d_dtable, d_n_dev);
        PERF_LAUNCH_CHECK();
    }
    return PERF_OK;
}

int perf_weights_from_density(const float* d_t_starts, const float* d_t_ends, const float* d_sigmas,
                              const int64_t* d_ray_indices, uint64_t N, uint64_t n_rays,
                              float* d_weights, float* d_trans, float* d_alphas, void* stream)
{
    PERF_CHECK_ARG(d_t_starts && d_t_ends && d_sigmas && d_ray_indices, "NULL pointer");
    if (N == 0 || n_rays == 0) return PERF_OK;
    weights_from_density_kernel<<<blocks_for(n_rays * 32, 256), 256, 0, S(stream)>>>(
        d_t_starts, d_t_ends, d_sigmas, d_ray_indices, N, n_rays, d_weights, d_trans, d_alphas);
    PERF_LAUNCH_CHECK();
    return PERF_OK;
}

int perf_weights_from_density_bwd(const float* d_t_starts, const float* d_t_ends, const float* d_sigmas,
                                  const int64_t* d_ray_indices, uint64_t N, uint64_t n_rays,
                                  const float* d_weights, const float* d_trans,
                                  const float* d_grad_weights, const float* d_grad_trans, float* d_grad_sigmas, void* stream)
{
    (void)d_sigmas;
    PERF_CHECK_ARG(d_t_starts && d_t_ends && d_ray_indices && d_weights && d_trans && d_grad_weights && d_grad_sigmas, "NULL pointer");
    if (N == 0 || n_rays == 0) return PERF_OK;
    weights_from_density_bwd_kernel<<<blocks_for(n_rays * 32, 256), 256, 0, S(stream)>>>(
        d_t_starts, d_t_ends, d_ray_indices, N, n_rays, d_weights, d_trans, d_grad_weights, d_grad_trans, d_grad_sigmas);
    PERF_LAUNCH_CHECK();
    return PERF_OK;
}

int perf_accumulate_along_rays(const float* d_weights, const float* d_values, int D, const int64_t* d_ray_indices,
                               uint64_t N, uint64_t n_rays, float* d_out, void* stream)
{
    PERF_CHECK_ARG(d_weights && d_ray_indices && d_out, "NULL pointer");
    PERF_CHECK_ARG(D >= 1 && D <= 64 && (d_values || D == 1), "bad D=%d", D);
    if (n_rays == 0) return PERF_OK;
    accumulate_along_rays_kernel<<<blocks_for(n_rays * 32, 256), 256, 0, S(stream)>>>(
        d_weights, d_values, D, d_ray_indices, N, n_rays, d_out);
    PERF_LAUNCH_CHECK();
    return PERF_OK;
}

int perf_adam_step(float* d_params, const float* d_grads, float* d_exp_avg, float* d_exp_avg_sq, void* d_params_half,
                   uint64_t n, float lr, float beta1, float beta2, float eps, uint32_t step, float grad_scale, void* stream)
{
    PERF_CHECK_ARG(d_params && d_grads && d_exp_avg && d_exp_avg_sq, "NULL pointer");
    PERF_CHECK_ARG(step >= 1, "step is 1-based");
    if (n == 0) return PERF_OK;
    const float bc1 = 1.0f - powf(beta1, (float)step);
    const float bc2_sqrt = sqrtf(1.0f - powf(beta2, (float)step));
    const int vec = adam_vec_ok(d_params, d_grads, d_exp_avg, d_exp_avg_sq, d_params_half) ? 1 : 0;
    const uint64_t threads = vec ? (n / 4 > n % 4 ? n / 4 : n % 4) : n;
    adam_kernel<<<blocks_for(threads ? threads : 1, 256), 256, 0, S(stream)>>>(d_params, d_grads, d_exp_avg, d_exp_avg_sq, (__half*)d_params_half,
                                                           n, lr, beta1, beta2, eps, bc1, bc2_sqrt, grad_scale, nullptr, vec);
    PERF_LAUNCH_CHECK();
    return PERF_OK;
}

int perf_set_scalars(float* d_dst, const float* h_values, int n, void* stream)
{
    PERF_CHECK_ARG(d_dst && h_values && n >= 1 && n <= 8, "perf_set_scalars: need 1..8 values");
    Scalars8 s; for (int i = 0; i < 8; ++i) s.v[i] = i < n ? h_values[i] : 0.f;   // by-value: no host-buffer lifetime issues
    set_scalars_kernel<<<1, 32, 0, S(stream)>>>(d_dst, s, n);
    PERF_LAUNCH_CHECK();
    return PERF_OK;
}

int perf_adam_step_dev(float* d_params, const float* d_grads, float* d_exp_avg, float* d_exp_avg_sq, void* d_params_half,
                       uint64_t n, const float* d_hyper, float beta1, float beta2, float eps, float grad_scale, void* stream)
{
    PERF_CHECK_ARG(d_params && d_grads && d_exp_avg && d_exp_avg_sq && d_hyper, "NULL pointer");
    if (n == 0) return PERF_OK;
    const int vec = adam_vec_ok(d_params, d_grads, d_exp_avg, d_exp_avg_sq, d_params_half) ? 1 : 0;
    const uint64_t threads = vec ? (n / 4 > n % 4 ? n / 4 : n % 4) : n;
    adam_kernel<<<blocks_for(threads ? threads : 1, 256), 256, 0, S(stream)>>>(d_params, d_grads, d_exp_avg, d_exp_avg_sq, (__half*)d_params_half,
                                                           n, 0.f, beta1, beta2, eps, 1.f, 1.f, grad_scale, d_hyper, vec);
    PERF_LAUNCH_CHECK();
    return PERF_OK;
}

#pragma GCC visibility pop
}  // extern "C"
