// texture_fill.cu -- pull-push fill of a texture's unused texels: each unused texel takes the rounded mean of the used texels
// of the smallest aligned power-of-two block (side >= 2) around it that holds any.  Three passes over 32 x 32 texel tiles:
// pull (per tile, the block sums of levels 1-5 in shared memory; only the level-5 record goes to the workspace), up (levels
// 6 .. log2 T from the level-5 records, 32 x 32 records per CTA, at most two launches) and push (per tile, levels 1-5 again,
// then each unused texel walks up to its first non-empty block, reading levels >= 6 from the workspace).  Integer arithmetic
// only and no atomics, so the result does not depend on execution order, and the host build of tests/texture_fill_harness.py
// (-DPERF_HOST_HARNESS: each CTA's phases run over host arrays in a serial loop) agrees bit for bit.
// Rule: perfb200.h (perf_texture_fill); restated in numpy in tests/texture_fill_oracle.py.
#include "common.cuh"

namespace perf {

constexpr int FILL_TILE = 32;                   // texels (or records) per CTA side: levels 1-5 inside a CTA
constexpr int FILL_THREADS = 256;               // one per level-1 block of a tile; 192 load the image rows, 64 the mask rows
constexpr int FILL_RECS = 256 + 64 + 16 + 4 + 1;

struct FillRec { int64_t n, s[3]; };            // used texels of a block and their channel sums

struct FillTile {                               // a CTA's shared memory
    uint4 img[FILL_TILE * 6];                   // 32 rows of 96 bytes
    uint4 msk[FILL_TILE * 2];                   // 32 rows of 32 bytes
    FillRec rec[FILL_RECS];                     // local levels 1-5, level r at fill_off(r), row-major
};

struct FillArgs {
    const uint8_t* image; const uint8_t* used; uint8_t* out;
    FillRec* ws;                                // levels 5 .. L, level l at fill_ws_off(T, l), (T >> l)^2 records row-major
    int32_t size, levels;                       // T, L = log2 T
    int32_t k;                                  // up: the input level
    uint8_t empty[3];
};

__host__ __device__ __forceinline__ int fill_log2(int v)
{
    int l = 0;
    while ((2 << l) <= v) ++l;
    return l;
}

__host__ __device__ __forceinline__ int fill_off(int r)
{
    int o = 0;
    for (int q = 1; q < r; ++q) o += (FILL_TILE >> q) * (FILL_TILE >> q);
    return o;
}

__host__ __device__ __forceinline__ int64_t fill_ws_off(int32_t T, int l)
{
    int64_t o = 0;
    for (int q = 5; q < l; ++q) o += (int64_t)(T >> q) * (T >> q);
    return o;
}

__host__ __device__ __forceinline__ void fill_add(FillRec& a, const FillRec& b)
{
    a.n += b.n; a.s[0] += b.s[0]; a.s[1] += b.s[1]; a.s[2] += b.s[2];
}

// Thread t of tile c: one 16-byte piece of the tile's image rows (t < 192) or mask rows (t >= 192).
__host__ __device__ __forceinline__ void fill_load(const FillArgs& a, FillTile& s, int64_t c, int t)
{
    const int64_t nt = a.size / FILL_TILE, tx = c % nt, ty = c / nt;
    if (t < 6 * FILL_TILE) {
        const int64_t row = ty * FILL_TILE + t / 6;
        s.img[t] = *(const uint4*)(a.image + 3 * (row * a.size + tx * FILL_TILE) + 16 * (t % 6));
    } else {
        const int u = t - 6 * FILL_TILE;
        const int64_t row = ty * FILL_TILE + u / 2;
        s.msk[u] = *(const uint4*)(a.used + row * a.size + tx * FILL_TILE + 16 * (u % 2));
    }
}

// Level 1 from the texels: thread t sums the used texels of the 2 x 2 block (t & 15, t >> 4) of the tile.
__host__ __device__ __forceinline__ void fill_texels(FillTile& s, int t)
{
    const uint8_t* img = (const uint8_t*)s.img;
    const uint8_t* msk = (const uint8_t*)s.msk;
    const int bx = t & 15, by = t >> 4;
    FillRec r = {0, {0, 0, 0}};
    for (int dy = 0; dy < 2; ++dy)
        for (int dx = 0; dx < 2; ++dx) {
            const int y = 2 * by + dy, x = 2 * bx + dx;
            if (msk[y * FILL_TILE + x]) {
                r.n += 1;
                for (int ch = 0; ch < 3; ++ch) r.s[ch] += img[3 * (y * FILL_TILE + x) + ch];
            }
        }
    s.rec[t] = r;
}

// Local level 1 of an up CTA from the input level k (side n = T >> k; the CTA covers a w x w square of it, w = min(32, n)):
// thread t < (w / 2)^2 sums four level-k records of the workspace.
__host__ __device__ __forceinline__ void fill_gather(const FillArgs& a, FillTile& s, int64_t c, int t)
{
    const int64_t n = a.size >> a.k, w = n < FILL_TILE ? n : FILL_TILE, h = w / 2, nc = n / w, cx = c % nc, cy = c / nc;
    if (t >= h * h) return;
    const int64_t x = t % h, y = t / h;
    const FillRec* in = a.ws + fill_ws_off(a.size, a.k);
    FillRec r = {0, {0, 0, 0}};
    for (int dy = 0; dy < 2; ++dy)
        for (int dx = 0; dx < 2; ++dx) fill_add(r, in[(cy * w + 2 * y + dy) * n + cx * w + 2 * x + dx]);
    s.rec[t] = r;
}

// Local level r >= 2 of a CTA of side w: thread t < (w >> r)^2 sums its four children of level r - 1.
__host__ __device__ __forceinline__ void fill_reduce(FillTile& s, int w, int r, int t)
{
    const int m = w >> r;
    if (t >= m * m) return;
    const int x = t % m, y = t / m;
    const FillRec* lo = s.rec + fill_off(r - 1);
    FillRec o = {0, {0, 0, 0}};
    for (int dy = 0; dy < 2; ++dy)
        for (int dx = 0; dx < 2; ++dx) fill_add(o, lo[(2 * y + dy) * (2 * m) + 2 * x + dx]);
    s.rec[fill_off(r) + t] = o;
}

// Record t of local level r of CTA c (side w, over input level k) to level k + r of the workspace.
__host__ __device__ __forceinline__ void fill_store(const FillArgs& a, const FillTile& s, int64_t c, int w, int r, int t)
{
    const int m = w >> r;
    if (t >= m * m) return;
    const int64_t n = a.size >> a.k, nc = n / w, cx = c % nc, cy = c / nc, nl = n >> r;
    a.ws[fill_ws_off(a.size, a.k + r) + (cy * m + t / m) * nl + cx * m + t % m] = s.rec[fill_off(r) + t];
}

__host__ __device__ __forceinline__ uint8_t fill_mean(const FillRec& r, int ch)
{
    return (uint8_t)((2 * r.s[ch] + r.n) / (2 * r.n));
}

// Thread t of tile c: the colour of the unused texels of its level-1 block (bx, by) = (t & 15, t >> 4), all of which share
// their ancestors: the mean of the first block with used texels, local levels 1-5, then levels 6 .. L of the workspace,
// else `empty`.  Written into the tile's image.
__host__ __device__ __forceinline__ void fill_push(const FillArgs& a, FillTile& s, int64_t c, int t)
{
    const int bx = t & 15, by = t >> 4;
    const int64_t nt = a.size / FILL_TILE, tx = c % nt, ty = c / nt;
    const FillRec* hit = nullptr;
    for (int r = 1; r <= 5 && !hit; ++r) {
        const FillRec* q = s.rec + fill_off(r) + (by >> (r - 1)) * (16 >> (r - 1)) + (bx >> (r - 1));
        if (q->n > 0) hit = q;
    }
    for (int l = 6; l <= a.levels && !hit; ++l) {
        const FillRec* q = a.ws + fill_ws_off(a.size, l) + (ty >> (l - 5)) * (nt >> (l - 5)) + (tx >> (l - 5));
        if (q->n > 0) hit = q;
    }
    uint8_t col[3];
    for (int ch = 0; ch < 3; ++ch) col[ch] = hit ? fill_mean(*hit, ch) : a.empty[ch];
    uint8_t* img = (uint8_t*)s.img;
    const uint8_t* msk = (const uint8_t*)s.msk;
    for (int dy = 0; dy < 2; ++dy)
        for (int dx = 0; dx < 2; ++dx) {
            const int y = 2 * by + dy, x = 2 * bx + dx;
            if (!msk[y * FILL_TILE + x])
                for (int ch = 0; ch < 3; ++ch) img[3 * (y * FILL_TILE + x) + ch] = col[ch];
        }
}

__host__ __device__ __forceinline__ void fill_write(const FillArgs& a, const FillTile& s, int64_t c, int t)
{
    if (t >= 6 * FILL_TILE) return;
    const int64_t nt = a.size / FILL_TILE, tx = c % nt, ty = c / nt, row = ty * FILL_TILE + t / 6;
    *(uint4*)(a.out + 3 * (row * a.size + tx * FILL_TILE) + 16 * (t % 6)) = s.img[t];
}

enum { FILL_PULL, FILL_UP, FILL_PUSH };

// Phase p of CTA c, thread t; the phases of a CTA are separated by barriers.  Pull and push: 0 load, 1 level 1, 2-5 levels
// 2-5, then pull 6 store level 5, push 6 fill, 7 write.  Up: 0 local level 1, 1 .. R - 1 levels 2 .. R, then R + r - 1
// stores local level r (r = 1 .. R, R = log2 w).
template <int S>
__host__ __device__ __forceinline__ void fill_phase(const FillArgs& a, FillTile& s, int64_t c, int p, int t)
{
    if (S == FILL_UP) {
        const int64_t n = a.size >> a.k;
        const int w = (int)(n < FILL_TILE ? n : FILL_TILE), R = fill_log2(w);
        if (p == 0) fill_gather(a, s, c, t);
        else if (p < R) fill_reduce(s, w, p + 1, t);
        else fill_store(a, s, c, w, p - R + 1, t);
        return;
    }
    if (p == 0) fill_load(a, s, c, t);
    else if (p == 1) fill_texels(s, t);
    else if (p <= 5) fill_reduce(s, FILL_TILE, p, t);
    else if (S == FILL_PULL) fill_store(a, s, c, FILL_TILE, 5, t);
    else if (p == 6) fill_push(a, s, c, t);
    else fill_write(a, s, c, t);
}

template <int S>
__host__ __device__ __forceinline__ int fill_phases(const FillArgs& a)
{
    if (S == FILL_PULL) return 7;
    if (S == FILL_PUSH) return 8;
    const int64_t n = a.size >> a.k;
    const int w = (int)(n < FILL_TILE ? n : FILL_TILE);
    return 2 * (fill_log2(w));
}

template <int S>
__global__ void __launch_bounds__(FILL_THREADS) fill_kernel(const FillArgs a)
{
    __shared__ FillTile s;
    const int np = fill_phases<S>(a);
    for (int p = 0; p < np; ++p) {
        fill_phase<S>(a, s, blockIdx.x, p, threadIdx.x);
        __syncthreads();
    }
}

// The product library launches the kernel; the test harness build runs the same phases over host arrays.
template <int S>
static int fill_run(const FillArgs& a, int64_t ctas, void* stream)
{
#ifdef PERF_HOST_HARNESS
    (void)stream;
    static FillTile s;
    const int np = fill_phases<S>(a);
    for (int64_t c = 0; c < ctas; ++c)
        for (int p = 0; p < np; ++p)
            for (int t = 0; t < FILL_THREADS; ++t) fill_phase<S>(a, s, c, p, t);
#else
    fill_kernel<S><<<(unsigned)ctas, FILL_THREADS, 0, (cudaStream_t)stream>>>(a);
    PERF_LAUNCH_CHECK();
#endif
    return PERF_OK;
}

}  // namespace perf

using namespace perf;

static bool fill_size_ok(int size)
{
    return size >= 256 && size <= 16384 && (size & (size - 1)) == 0;
}

extern "C" {
#pragma GCC visibility push(default)

uint64_t perf_texture_fill_workspace_bytes(int size)
{
    if (!fill_size_ok(size)) return 0;
    return (uint64_t)sizeof(FillRec) * (uint64_t)fill_ws_off(size, fill_log2(size) + 1);
}

int perf_texture_fill(const uint8_t* d_image, const uint8_t* d_used, int size, const uint8_t* h_empty, void* d_workspace,
                      uint64_t workspace_bytes, uint8_t* d_out, void* stream)
{
    PERF_CHECK_ARG(fill_size_ok(size), "texture size %d: needs a power of two in [256, 16384]", size);
    PERF_CHECK_ARG(d_image && d_used && h_empty && d_workspace && d_out, "NULL pointer");
    PERF_CHECK_ARG(((uintptr_t)d_image | (uintptr_t)d_used | (uintptr_t)d_out | (uintptr_t)d_workspace) % 16 == 0,
                   "image, used mask, output and workspace must be 16-byte aligned");
    PERF_CHECK_ARG(workspace_bytes >= perf_texture_fill_workspace_bytes(size), "workspace of %llu bytes, needs %llu",
                   (unsigned long long)workspace_bytes, (unsigned long long)perf_texture_fill_workspace_bytes(size));
    FillArgs a;
    memset(&a, 0, sizeof(a));
    a.image = d_image; a.used = d_used; a.out = d_out; a.ws = (FillRec*)d_workspace;
    a.size = size; a.levels = fill_log2(size);
    for (int ch = 0; ch < 3; ++ch) a.empty[ch] = h_empty[ch];
    const int64_t tiles = (int64_t)(size / FILL_TILE) * (size / FILL_TILE);
    int rc = fill_run<FILL_PULL>(a, tiles, stream); if (rc) return rc;
    for (a.k = 5; a.k < a.levels; a.k += 5) {
        const int64_t n = size >> a.k, w = n < FILL_TILE ? n : FILL_TILE;
        rc = fill_run<FILL_UP>(a, (n / w) * (n / w), stream); if (rc) return rc;
    }
    a.k = 0;
    return fill_run<FILL_PUSH>(a, tiles, stream);
}

#pragma GCC visibility pop
}
