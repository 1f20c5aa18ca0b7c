// occ.cu -- occupancy-grid interval sampler (nerfacc OccGridEstimator.sampling semantics for
// levels=1, cone_angle=0; SURVEY.md section 8f row 1; call site modules/scene/nerf_renderer.py:145-155).
// Rule (restated in oracle/occ_sampler.py): lattice t_k = near + (k + u_r) * step; the interval
// [t_k, t_k + step) is emitted when its midpoint lies inside the ray/aabb overlap and in an occupied
// cell.  Two passes (count, write) around an exclusive scan of the per-ray counts done by the caller.
#include "common.cuh"

namespace perf {

constexpr uint32_t PERF_OCC_MAX_STEPS = 1u << 22;      // lattice points one ray may visit (PeRF: 1.5 / 5e-4 = 3000)
constexpr int PERF_OCC_MASK_WORDS = 4;

struct OccArgs {
    const uint8_t* binaries; int rx, ry, rz;
    float amin[3], aext[3], amax[3];
    const float *rays_o, *rays_d, *jitter;
    uint64_t R; float near, far, step;
    int32_t* counts; const int64_t* offsets;
    int64_t* ray_indices; float *t_starts, *t_ends;
    int64_t capacity;            // write pass: samples at positions >= capacity are dropped (0 = no limit)
    uint32_t pieces;             // every ray's lattice range is cut into `pieces` consecutive parts marched by different threads:
                                 // counts / offsets are indexed [ray * pieces + piece] (the packed output order is unchanged)
    uint32_t* masks;             // optional [R * pieces][PERF_OCC_MASK_WORDS]: bit j of a slot = lattice point (first index of the
                                 // piece + j) is a sample.  Written by the count pass; the write pass then only expands the bits
                                 // (no second march, no second read of the grid).  Needs <= 32 * PERF_OCC_MASK_WORDS points per piece.
};

// One ray.  __host__ __device__: tests/host_harness.py compiles this file with -DPERF_HOST_HARNESS into a separate
// test-only object and runs the same body over host arrays against oracle/occ_sampler.py.
template <bool WRITE>
__host__ __device__ __forceinline__ void occ_march_ray(const OccArgs& a, uint64_t ray, uint32_t piece = 0)
{
    const uint32_t P = a.pieces ? a.pieces : 1u;
    const uint64_t slot = ray * P + piece;
    uint32_t bits[PERF_OCC_MASK_WORDS] = {0u, 0u, 0u, 0u};
    const bool expand = WRITE && a.masks != nullptr;          // write pass with masks: expand the count pass's bits, do not march
    const float o[3] = {a.rays_o[3 * ray], a.rays_o[3 * ray + 1], a.rays_o[3 * ray + 2]};
    const float d[3] = {a.rays_d[3 * ray], a.rays_d[3 * ray + 1], a.rays_d[3 * ray + 2]};
    float tn = -INFINITY, tf = INFINITY;
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        const float inv = PERF_FDIV_RN(1.0f, fabsf(d[i]) < 1e-12f ? 1e-12f : d[i]);
        const float t0 = PERF_FMUL_RN(PERF_FSUB_RN(a.amin[i], o[i]), inv), t1 = PERF_FMUL_RN(PERF_FSUB_RN(a.amax[i], o[i]), inv);
        tn = fmaxf(tn, fminf(t0, t1)); tf = fminf(tf, fmaxf(t0, t1));
    }
    tn = fmaxf(tn, a.near); tf = fminf(tf, a.far);
    const float u = a.jitter ? a.jitter[ray] : 0.f;
    const float half_step = PERF_FMUL_RN(0.5f, a.step);
    int64_t pos = WRITE ? a.offsets[slot] : 0;
    int32_t n = 0;
    if (tf >= tn) {
        // first lattice index whose midpoint can reach tn (minus a safety margin; exact test below)
        float kf = floorf((tn - a.near) / a.step - u - 0.5f) - 2.0f;
        uint32_t k = kf > 0.f ? (uint32_t)kf : 0u;
        // Bounded walk: at most the lattice points between tn and tf (+ margin).  A ray whose overlap with the box
        // is not bounded by the box (|d| ~ 0 with far_plane = 1e10, or a tiny step) would otherwise spin once
        // (float)k stops changing at 2^24; such a ray yields no samples.
        const float span = (tf - tn) / a.step;
        uint32_t k_end = span < (float)PERF_OCC_MAX_STEPS ? k + (uint32_t)span + 8u : k;
        if (P > 1) {                                           // this thread's part of [k, k_end): the same per-point tests, fewer of them
            const uint32_t per = (k_end - k + P - 1u) / P;
            const uint32_t lo = k + piece * per;
            k_end = (lo + per < k_end) ? lo + per : k_end;
            k = lo < k_end ? lo : k_end;
        }
        const uint32_t k_first = k;
        if (expand) {
            for (int j = 0; j < 32 * PERF_OCC_MASK_WORDS; ++j) {
                if ((a.masks[slot * PERF_OCC_MASK_WORDS + (j >> 5)] >> (j & 31)) & 1u) {
                    const uint32_t kk = k_first + (uint32_t)j;
                    const float ts = fixed_s_t(a.near, a.step, kk, u);
                    if (a.capacity == 0 || pos < a.capacity) { a.ray_indices[pos] = (int64_t)ray; a.t_starts[pos] = ts; a.t_ends[pos] = PERF_FADD_RN(ts, a.step); }
                    ++pos;
                }
            }
            k = k_end;                                         // skip the march below
        }
        for (; k < k_end; ++k) {
            const float ts = fixed_s_t(a.near, a.step, k, u);
            const float mid = PERF_FADD_RN(ts, half_step);
            if (mid > tf) break;
            if (mid < tn) continue;
            int c[3]; float pnt[3];
#pragma unroll
            for (int i = 0; i < 3; ++i) {
                const float p = PERF_FADD_RN(o[i], PERF_FMUL_RN(d[i], mid));
                pnt[i] = p;
                const int res = i == 0 ? a.rx : (i == 1 ? a.ry : a.rz);
                int ci = (int)floorf(PERF_FMUL_RN(to_unit(p, a.amin[i], a.aext[i]), (float)res));
                c[i] = ci < 0 ? 0 : (ci > res - 1 ? res - 1 : ci);
            }
            if (a.binaries[((int64_t)c[0] * a.ry + c[1]) * a.rz + c[2]]) {
                if (WRITE) {
                    if (a.capacity == 0 || pos < a.capacity) { a.ray_indices[pos] = (int64_t)ray; a.t_starts[pos] = ts; a.t_ends[pos] = PERF_FADD_RN(ts, a.step); }
                    ++pos;
                } else if (a.masks) {
                    const uint32_t j = k - k_first;            // < 32 * PERF_OCC_MASK_WORDS (checked on the host)
                    bits[j >> 5] |= 1u << (j & 31);
                }
                ++n;
            } else {
                // EMPTY cell: every lattice point whose midpoint stays inside it is rejected by the same test, so jump to just
                // before the cell's exit instead of visiting them one by one (PeRF: 15.6 lattice steps per cell of the 256^3
                // grid, 98 % of the cells empty).  The exit distance is the nearest of the three slab crossings ahead of `mid`;
                // the jump keeps a margin of 3 steps (>> the fp32 error of the slab arithmetic), and the points after it go
                // through the exact per-point test above again, so the emitted set is unchanged (tests/test_occ_host.py).
                float t_exit = INFINITY;
#pragma unroll
                for (int i = 0; i < 3; ++i) {
                    const int res = i == 0 ? a.rx : (i == 1 ? a.ry : a.rz);
                    const float cell = a.aext[i] / (float)res;
                    if (d[i] > 1e-9f)       t_exit = fminf(t_exit, mid + (a.amin[i] + (float)(c[i] + 1) * cell - pnt[i]) / d[i]);
                    else if (d[i] < -1e-9f) t_exit = fminf(t_exit, mid + (a.amin[i] + (float)c[i] * cell - pnt[i]) / d[i]);
                }
                if (t_exit < INFINITY) {
                    const float kf2 = floorf((t_exit - a.near) / a.step - u - 0.5f) - 3.0f;
                    if (kf2 > (float)k && kf2 < (float)k_end) k = (uint32_t)kf2;          // the loop's ++k follows
                }
            }
        }
    }
    if (!WRITE) {
        a.counts[slot] = n;
        if (a.masks) { for (int w = 0; w < PERF_OCC_MASK_WORDS; ++w) a.masks[slot * PERF_OCC_MASK_WORDS + w] = bits[w]; }
    }
}

template <bool WRITE>
__global__ void __launch_bounds__(128) occ_march_kernel(const OccArgs a)
{
    const uint64_t ray = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (ray < a.R) occ_march_ray<WRITE>(a, ray, blockIdx.y);
}

}  // namespace perf

using namespace perf;

static int fill(OccArgs& a, const uint8_t* bin, const int* res3, const float* aabb6, const float* o, const float* d, const float* jit,
                uint64_t R, float near, float far, float step, uint32_t pieces = 1)
{
    PERF_CHECK_ARG(bin && res3 && aabb6 && o && d, "NULL pointer");
    PERF_CHECK_ARG(res3[0] > 0 && res3[1] > 0 && res3[2] > 0 && step > 0.f && far > near, "bad occupancy sampling arguments");
    memset(&a, 0, sizeof(a));
    a.binaries = bin; a.rx = res3[0]; a.ry = res3[1]; a.rz = res3[2];
    for (int i = 0; i < 3; ++i) { a.amin[i] = aabb6[i]; a.amax[i] = aabb6[3 + i]; a.aext[i] = aabb6[3 + i] - aabb6[i]; }
    a.rays_o = o; a.rays_d = d; a.jitter = jit; a.R = R; a.near = near; a.far = far; a.step = step;
    PERF_CHECK_ARG(pieces >= 1 && pieces <= 1024, "pieces=%u not in [1,1024]", pieces);
    a.pieces = pieces;
    return PERF_OK;
}
// masks are usable when no piece can hold more lattice points than the mask has bits
static int check_masks(const OccArgs& a, const void* masks)
{
    if (!masks) return PERF_OK;
    PERF_CHECK_ARG((uintptr_t)masks % 4 == 0, "misaligned masks");
    const double max_points = ((double)a.far - (double)a.near) / (double)a.step + 16.0;
    PERF_CHECK_ARG(max_points / (double)a.pieces + 1.0 <= 32.0 * PERF_OCC_MASK_WORDS,
                   "sample masks need <= %d lattice points per piece: (far - near) / step / pieces = %.0f", 32 * PERF_OCC_MASK_WORDS, max_points / a.pieces);
    return PERF_OK;
}

extern "C" {
#pragma GCC visibility push(default)

int perf_occ_count(const uint8_t* d_binaries, const int* h_res3, const float* h_aabb6, const float* d_rays_o, const float* d_rays_d,
                   const float* d_jitter, uint64_t R, float near, float far, float step, uint32_t pieces, int32_t* d_counts, uint32_t* d_masks,
                   void* stream)
{
    OccArgs a; int rc = fill(a, d_binaries, h_res3, h_aabb6, d_rays_o, d_rays_d, d_jitter, R, near, far, step, pieces); if (rc) return rc;
    PERF_CHECK_ARG(d_counts, "NULL counts");
    rc = check_masks(a, d_masks); if (rc) return rc;
    a.counts = d_counts; a.masks = d_masks;
    if (R == 0) return PERF_OK;
    occ_march_kernel<false><<<dim3((unsigned)((R + 127) / 128), pieces), 128, 0, (cudaStream_t)stream>>>(a);
    PERF_LAUNCH_CHECK();
    return PERF_OK;
}

int perf_occ_write(const uint8_t* d_binaries, const int* h_res3, const float* h_aabb6, const float* d_rays_o, const float* d_rays_d,
                   const float* d_jitter, uint64_t R, float near, float far, float step, uint32_t pieces, const int64_t* d_offsets, uint64_t capacity,
                   const uint32_t* d_masks, int64_t* d_ray_indices, float* d_t_starts, float* d_t_ends, void* stream)
{
    OccArgs a; int rc = fill(a, d_binaries, h_res3, h_aabb6, d_rays_o, d_rays_d, d_jitter, R, near, far, step, pieces); if (rc) return rc;
    rc = check_masks(a, d_masks); if (rc) return rc;
    a.masks = const_cast<uint32_t*>(d_masks);
    PERF_CHECK_ARG(d_offsets && d_ray_indices && d_t_starts && d_t_ends, "NULL output");
    a.offsets = d_offsets; a.ray_indices = d_ray_indices; a.t_starts = d_t_starts; a.t_ends = d_t_ends; a.capacity = (int64_t)capacity;
    if (R == 0) return PERF_OK;
    occ_march_kernel<true><<<dim3((unsigned)((R + 127) / 128), pieces), 128, 0, (cudaStream_t)stream>>>(a);
    PERF_LAUNCH_CHECK();
    return PERF_OK;
}

#ifdef PERF_HOST_HARNESS
/* TEST HARNESS ONLY (never compiled into libperfb200.so): the per-ray body over HOST arrays.  pass 0 = count, 1 = write. */
int perf_host_occ_march(int pass, const uint8_t* h_binaries, const int* h_res3, const float* h_aabb6, const float* h_rays_o,
                        const float* h_rays_d, const float* h_jitter, uint64_t R, float near, float far, float step, uint32_t pieces,
                        int32_t* h_counts, const int64_t* h_offsets, int64_t* h_ray_indices, float* h_t_starts, float* h_t_ends, uint32_t* h_masks)
{
    OccArgs a; int rc = fill(a, h_binaries, h_res3, h_aabb6, h_rays_o, h_rays_d, h_jitter, R, near, far, step, pieces); if (rc) return rc;
    rc = check_masks(a, h_masks); if (rc) return rc;
    a.masks = h_masks;
    a.counts = h_counts; a.offsets = h_offsets; a.ray_indices = h_ray_indices; a.t_starts = h_t_starts; a.t_ends = h_t_ends;
    for (uint32_t pc = 0; pc < pieces; ++pc)
        for (uint64_t r = 0; r < R; ++r) { if (pass == 0) occ_march_ray<false>(a, r, pc); else occ_march_ray<true>(a, r, pc); }
    return PERF_OK;
}
#endif

#pragma GCC visibility pop
}
