// png.cu -- PNG encoder (8-bit RGB, no interlace) with all of the compression on the GPU.  Three launches in perf_png_compress
// and one in perf_png_write:
//   filter  (one CTA per row): the five PNG filters' costs, the cheapest filter's row into the filtered stream;
//   segment (one CTA per segment of whole rows, <= 65535 filtered bytes): runs, the closed-form token parse, the histogram,
//           length-limited Huffman codes, the dynamic block (or a stored one when that is shorter) written into shared memory
//           with word-wide ORs, the segment's Adler-32 sums and the CRC-32 of its IDAT chunk;
//   finish  (one CTA): file offsets of the chunks, the combined Adler-32, the file size, the last chunk's CRC over the trailer;
//   write   (one CTA per chunk, one more for the header and IEND): the file.
// Integer arithmetic only; the only atomics are integer adds and ORs, so the bytes do not depend on execution order, and the
// host build of tests/png_harness.py (-DPERF_HOST_HARNESS: each CTA's phases run over host arrays in a serial loop) agrees
// bit for bit.  Rule: perfb200.h (perf_png_*); the filter choice and the segment split restated in numpy in
// tests/png_oracle.py.
#include "common.cuh"

namespace perf {

constexpr int PNG_MAX_W = 21844;                // a filtered row, 1 + 3 W bytes, fits one stored block
constexpr int PNG_SEG_MAX = 65535;
constexpr int PNG_SLOT = 65544;                 // workspace bytes per segment: a stored segment (5 + 65535) rounded up to 8
constexpr int PNG_FILTER_THREADS = 256;
constexpr int PNG_THREADS = 1024;               // segment CTA: thread t parses filtered bytes [64 t, 64 t + 64)
constexpr int PNG_CHUNK = 64;
constexpr int PNG_LITLEN = 286;
constexpr uint32_t PNG_ADLER_MOD = 65521;

struct PngSeg {                                 // per segment, written by the segment CTA (off by the finish CTA)
    uint32_t n;                                 // filtered bytes
    uint32_t m;                                 // compressed bytes (the deflate blocks, without the zlib header or trailer)
    uint32_t crc;                               // CRC-32 of the IDAT chunk (type and data; the last one with the trailer after finish)
    uint32_t s1, s2;                            // Adler-32 sums of the segment from a = b = 0
    uint32_t pad;
    uint64_t off;                               // file offset of the chunk
};

struct PngHead { uint64_t file_bytes; uint32_t adler; uint32_t pad; };

struct PngArgs {
    const uint8_t* image; uint8_t* filt; uint8_t* slots; PngSeg* segs; PngHead* head; uint8_t* out;
    int32_t H, W, rows;                         // rows per segment
    int64_t L;                                  // filtered row bytes, 1 + 3 W
    int64_t S;                                  // segments
};

__host__ __device__ __forceinline__ void png_inc(uint32_t* p)
{
#ifdef __CUDA_ARCH__
    atomicAdd(p, 1u);
#else
    ++*p;
#endif
}

// ---------------------------------------------------------------- CRC-32 (the PNG / zlib polynomial, reflected)
__host__ __device__ __forceinline__ uint32_t png_crc_bytes(uint32_t crc, const uint8_t* p, int64_t n)
{
    crc = ~crc;
    for (int64_t i = 0; i < n; ++i) {
        crc ^= p[i];
        for (int k = 0; k < 8; ++k) crc = (crc >> 1) ^ (0xEDB88320u & (0u - (crc & 1u)));
    }
    return ~crc;
}
// a * b modulo the polynomial (bit 31 = x^0)
__host__ __device__ __forceinline__ uint32_t png_mulmodp(uint32_t a, uint32_t b)
{
    uint32_t p = 0;
    for (uint32_t m = 1u << 31; m; m >>= 1) {
        if (a & m) p ^= b;
        b = (b & 1u) ? (b >> 1) ^ 0xEDB88320u : b >> 1;
    }
    return p;
}
// x^(2^k) modulo the polynomial
__host__ __device__ __forceinline__ uint32_t png_x2n(int k)
{
    const uint32_t tab[32] = {
        0x40000000, 0x20000000, 0x08000000, 0x00800000, 0x00008000, 0xedb88320, 0xb1e6b092, 0xa06a2517, 0xed627dae, 0x88d14467,
        0xd7bbfe6a, 0xec447f11, 0x8e7ea170, 0x6427800e, 0x4d47bae0, 0x09fe548f, 0x83852d0f, 0x30362f1a, 0x7b5a9cc3, 0x31fec169,
        0x9fec022a, 0x6c8dedc4, 0x15d6874d, 0x5fde7a4e, 0xbad90e37, 0x2e4e5eef, 0x4eaba214, 0xa8a472c0, 0x429a969e, 0x148d302a,
        0xc40ba6d0, 0xc4e22c3c};
    return tab[k & 31];
}
// CRC-32 of A || B from crc(A), crc(B) and |B| (bytes): crc(A) x^(8 |B|) + crc(B)
__host__ __device__ __forceinline__ uint32_t png_crc_combine(const uint32_t* x2n, uint32_t a, uint32_t b, int64_t nb)
{
    uint32_t op = 1u << 31;
    for (int k = 3; nb; nb >>= 1, ++k)
        if (nb & 1) op = png_mulmodp(x2n[k & 31], op);
    return png_mulmodp(op, a) ^ b;
}

// ---------------------------------------------------------------- filter: one CTA per row
struct PngFilterSmem { int32_t cost[5][PNG_FILTER_THREADS]; int32_t type; };

__host__ __device__ __forceinline__ int png_paeth(int a, int b, int c)
{
    const int p = a + b - c, pa = p > a ? p - a : a - p, pb = p > b ? p - b : b - p, pc = p > c ? p - c : c - p;
    return (pa <= pb && pa <= pc) ? a : (pb <= pc ? b : c);
}

// Residual byte of filter f at byte i of row y.
__host__ __device__ __forceinline__ uint8_t png_residual(const PngArgs& a, int64_t y, int64_t i, int f)
{
    const int64_t stride = 3 * (int64_t)a.W;
    const uint8_t* row = a.image + y * stride;
    const int x = row[i];
    const int l = i >= 3 ? row[i - 3] : 0;
    const int u = y > 0 ? row[i - stride] : 0;
    const int ul = (y > 0 && i >= 3) ? row[i - stride - 3] : 0;
    int pred = 0;
    if (f == 1) pred = l;
    else if (f == 2) pred = u;
    else if (f == 3) pred = (l + u) >> 1;
    else if (f == 4) pred = png_paeth(l, u, ul);
    return (uint8_t)(x - pred);
}

__host__ __device__ __forceinline__ void png_filter_phase(const PngArgs& a, PngFilterSmem& s, int64_t y, int p, int t)
{
    const int64_t n = 3 * (int64_t)a.W;
    if (p == 0) {
        int32_t c[5] = {0, 0, 0, 0, 0};
        for (int64_t i = t; i < n; i += PNG_FILTER_THREADS)
            for (int f = 0; f < 5; ++f) {
                const int r = (int8_t)png_residual(a, y, i, f);
                c[f] += r < 0 ? -r : r;
            }
        for (int f = 0; f < 5; ++f) s.cost[f][t] = c[f];
    } else if (p == 1) {
        if (t < 5) {
            int32_t c = 0;
            for (int j = 0; j < PNG_FILTER_THREADS; ++j) c += s.cost[t][j];
            s.cost[t][0] = c;
        }
    } else if (p == 2) {
        if (t == 0) {
            int best = 0;
            for (int f = 1; f < 5; ++f)
                if (s.cost[f][0] < s.cost[best][0]) best = f;
            s.type = best;
        }
    } else {
        uint8_t* out = a.filt + y * a.L;
        if (t == 0) out[0] = (uint8_t)s.type;
        for (int64_t i = t; i < n; i += PNG_FILTER_THREADS) out[1 + i] = png_residual(a, y, i, s.type);
    }
}
constexpr int PNG_FILTER_PHASES = 4;

// ---------------------------------------------------------------- segment: one CTA per segment
struct PngSmem {
    uint32_t out[PNG_SLOT / 4];                 // the segment's deflate bytes, built with ORs
    uint8_t in[PNG_SEG_MAX + 1];                // its filtered bytes
    uint32_t hist[PNG_LITLEN];                  // literal / length symbol counts
    uint16_t code[PNG_LITLEN];                  // bit-reversed canonical codes
    uint8_t len[PNG_LITLEN];
    int32_t sorted[PNG_LITLEN];                 // the used symbols by (count, symbol)
    uint32_t nused;
    // Huffman construction scratch of thread 0 (2 n - 1 nodes)
    int32_t weight[2 * PNG_LITLEN], parent[2 * PNG_LITLEN], depth[2 * PNG_LITLEN];
    int32_t blc[2 * PNG_LITLEN];
    // the code-length code: the run-length list of the lengths and its code
    uint8_t rle_sym[PNG_LITLEN + 2], rle_ext[PNG_LITLEN + 2];
    int32_t n_rle, hlit, hclen;
    uint8_t cl_len[19]; uint16_t cl_code[19];
    int64_t hdr_bits, tok_bits;
    int32_t stored, m;
    // per-thread partials and their group (32 threads) aggregates
    int32_t fb[PNG_THREADS], lb[PNG_THREADS], rs0[PNG_THREADS], re1[PNG_THREADS];
    int64_t bits[PNG_THREADS];
    uint32_t s1[PNG_THREADS]; uint64_t s2[PNG_THREADS];
    uint32_t crc[PNG_THREADS];
    int32_t gfb[32], glb[32], gpre[32], gsuf[32];
    int64_t gbits[32], gbpre[32];
    uint32_t seg_s1, seg_s2;
    uint32_t x2n[32];
};

__host__ __device__ __forceinline__ void png_len_sym(int L, int& sym, int& ext, int& ev)
{
    if (L == 258) { sym = 285; ext = 0; ev = 0; return; }
    const int l = L - 3;
    if (l < 8) { sym = 257 + l; ext = 0; ev = 0; return; }
    int lg = 3;
    while ((2 << lg) <= l) ++lg;
    ext = lg - 2;
    sym = 257 + 4 * (ext + 1) + ((l >> ext) - 4);
    ev = l & ((1 << ext) - 1);
}

// A word-aligned 64-bit accumulator over the shared output: one OR per 32 bits.
struct PngBits {
    uint32_t* out; int64_t base; uint64_t acc; int fill;
    __host__ __device__ __forceinline__ PngBits(uint32_t* o, int64_t pos) : out(o), base(pos & ~(int64_t)31), acc(0), fill((int)(pos & 31)) {}
    __host__ __device__ __forceinline__ void put(uint32_t v, int nb)
    {
        acc |= (uint64_t)v << fill;
        fill += nb;
        if (fill >= 32) {
            or_u32(out + (base >> 5), (uint32_t)acc);
            acc >>= 32; fill -= 32; base += 32;
        }
    }
    __host__ __device__ __forceinline__ void flush()
    {
        if (fill > 0) or_u32(out + (base >> 5), (uint32_t)acc);
    }
};

// The tokens of thread t's bytes [64 t, 64 t + 64) of the segment: mode 0 counts the symbols, 1 returns the bits they take,
// 2 writes them from bit `pos`.  Run [rs, re) of equal bytes: rs literal, then matches of min(258, rest) at distance 1 while
// at least 3 bytes remain, then 1-2 literals.
template <int MODE>
__host__ __device__ __forceinline__ int64_t png_walk(PngSmem& s, int n, int t, int64_t pos)
{
    const int i0 = PNG_CHUNK * t, i1 = i0 + PNG_CHUNK < n ? i0 + PNG_CHUNK : n;
    int64_t nbits = 0;
    PngBits w(s.out, pos);
    int rs = s.rs0[t], re = -1;
    for (int i = i0; i < i1; ++i) {
        if (i == 0 || s.in[i] != s.in[i - 1]) { rs = i; re = -1; }
        const int k = i - rs;
        int L = 0;                              // 0: literal, >= 3: match, -1: inside a match
        if (k > 0) {
            if (re < 0) {
                re = s.re1[t];
                for (int x = i + 1; x < i1; ++x)
                    if (s.in[x] != s.in[i]) { re = x; break; }
            }
            const int j = k - 1, r = re - rs - 1, full = (r / 258) * 258, rem = r - full;
            if (j < full) L = j % 258 == 0 ? 258 : -1;
            else if (j == full) L = rem >= 3 ? rem : 0;
            else L = rem >= 3 ? -1 : 0;
        }
        if (L < 0) continue;
        int sym = s.in[i], ext = 0, ev = 0;
        if (L) png_len_sym(L, sym, ext, ev);
        if (MODE == 0) {
            png_inc(s.hist + sym);
        } else {
            // the distance code: symbol 0 (distance 1) of a two-symbol code of length 1, code 0
            const int nb = s.len[sym] + ext + (L ? 1 : 0);
            if (MODE == 1) nbits += nb;
            else w.put((uint32_t)s.code[sym] | ((uint32_t)ev << s.len[sym]), nb);
        }
    }
    if (MODE == 2) w.flush();
    return nbits;
}

// Deterministic length-limited Huffman code lengths of the n >= 2 used symbols sym[0..n) sorted by (count, symbol): the
// two-queue Huffman tree (a leaf before an internal node of equal weight), its depths capped at `limit` and the Kraft sum
// restored (one leaf moves from the longest length below the limit that has one to the next length, with a leaf from the
// limit as its sibling, until the code is complete), then the lengths handed out longest first in sorted order.
__host__ __device__ __forceinline__ void png_huffman(PngSmem& s, const int32_t* sym, const uint32_t* cnt, int n, int limit,
                                                     uint8_t* len_out)
{
    int32_t* w = s.weight; int32_t* par = s.parent; int32_t* dep = s.depth; int32_t* bl = s.blc;
    // nodes: leaves 0 .. n-1, internal n .. 2n-2
    for (int i = 0; i < n; ++i) w[i] = (int32_t)cnt[sym[i]];
    int li = 0, ni = n;
    for (int k = n; k < 2 * n - 1; ++k) {
        int pick[2];
        for (int q = 0; q < 2; ++q) {
            if (li < n && (ni >= k || w[li] <= w[ni])) pick[q] = li++;
            else pick[q] = ni++;
        }
        w[k] = w[pick[0]] + w[pick[1]];
        par[pick[0]] = k; par[pick[1]] = k;
    }
    dep[2 * n - 2] = 0;
    for (int k = 2 * n - 3; k >= 0; --k) dep[k] = dep[par[k]] + 1;
    for (int l = 0; l <= (n > limit ? n : limit) + 1; ++l) bl[l] = 0;
    for (int i = 0; i < n; ++i) ++bl[dep[i] < limit ? dep[i] : limit];
    uint32_t total = 0;
    for (int l = 1; l <= limit; ++l) total += (uint32_t)bl[l] << (limit - l);
    while (total != (1u << limit)) {
        --bl[limit];
        for (int l = limit - 1; l > 0; --l)
            if (bl[l]) { --bl[l]; bl[l + 1] += 2; break; }
        --total;
    }
    int idx = 0;
    for (int l = limit; l >= 1; --l)
        for (int k = 0; k < bl[l]; ++k) len_out[sym[idx++]] = (uint8_t)l;
}

// Canonical (RFC 1951) codes of the lengths len[0..n), bit-reversed for LSB-first output.
__host__ __device__ __forceinline__ void png_codes(const uint8_t* len, int n, uint16_t* code)
{
    int bl[16] = {0}, next[16];
    for (int i = 0; i < n; ++i) ++bl[len[i]];
    bl[0] = 0;
    int c = 0;
    for (int l = 1; l < 16; ++l) { c = (c + bl[l - 1]) << 1; next[l] = c; }
    for (int i = 0; i < n; ++i) {
        if (!len[i]) { code[i] = 0; continue; }
        const int v = next[len[i]]++;
        int r = 0;
        for (int b = 0; b < len[i]; ++b) r |= ((v >> b) & 1) << (len[i] - 1 - b);
        code[i] = (uint16_t)r;
    }
}

__host__ __device__ __forceinline__ int png_cl_ext(int sym) { return sym == 16 ? 2 : sym == 17 ? 3 : sym == 18 ? 7 : 0; }

// The order in which the header lists the code-length code's lengths
__host__ __device__ __forceinline__ int png_cl_order(int i)
{
    return (uint8_t)"\x10\x11\x12\x00\x08\x07\x09\x06\x0a\x05\x0b\x04\x0c\x03\x0d\x02\x0e\x01\x0f"[i];
}

// Thread 0: the literal / length code, the run-length list of the code lengths, the code-length code and the header's bits.
__host__ __device__ __forceinline__ void png_tree(PngSmem& s)
{
    for (int i = 0; i < PNG_LITLEN; ++i) s.len[i] = 0;
    png_huffman(s, s.sorted, s.hist, (int)s.nused, 15, s.len);
    png_codes(s.len, PNG_LITLEN, s.code);
    int hlit = 257;
    for (int i = 257; i < PNG_LITLEN; ++i)
        if (s.len[i]) hlit = i + 1;
    s.hlit = hlit;
    // the lengths of the literal / length code, then the distance code's two lengths of 1
    const int total = hlit + 2;
    int nr = 0;
    for (int i = 0; i < total;) {
        const int v = i < hlit ? s.len[i] : 1;
        int run = 1;
        while (i + run < total && (i + run < hlit ? s.len[i + run] : 1) == v) ++run;
        i += run;
        if (v == 0) {
            while (run >= 3) {
                const int k = run >= 11 ? (run < 138 ? run : 138) : run;
                s.rle_sym[nr] = (uint8_t)(k >= 11 ? 18 : 17); s.rle_ext[nr++] = (uint8_t)(k >= 11 ? k - 11 : k - 3);
                run -= k;
            }
        } else {
            s.rle_sym[nr] = (uint8_t)v; s.rle_ext[nr++] = 0;
            --run;
            while (run >= 3) {
                const int k = run < 6 ? run : 6;
                s.rle_sym[nr] = 16; s.rle_ext[nr++] = (uint8_t)(k - 3);
                run -= k;
            }
        }
        for (; run > 0; --run) { s.rle_sym[nr] = (uint8_t)v; s.rle_ext[nr++] = 0; }
    }
    s.n_rle = nr;
    uint32_t ccnt[19] = {0};
    for (int i = 0; i < nr; ++i) ++ccnt[s.rle_sym[i]];
    // fewer than two used symbols: the lowest unused ones join with count 0, so that the code is complete
    int csym[19], cn = 0;
    for (int i = 0; i < 19; ++i)
        if (ccnt[i]) csym[cn++] = i;
    for (int i = 0; i < 19 && cn < 2; ++i)
        if (!ccnt[i]) csym[cn++] = i;
    // insertion sort by (count, symbol)
    for (int i = 1; i < cn; ++i)
        for (int j = i; j > 0 && (ccnt[csym[j]] < ccnt[csym[j - 1]] ||
                                  (ccnt[csym[j]] == ccnt[csym[j - 1]] && csym[j] < csym[j - 1])); --j) {
            const int tmp = csym[j]; csym[j] = csym[j - 1]; csym[j - 1] = tmp;
        }
    for (int i = 0; i < 19; ++i) s.cl_len[i] = 0;
    png_huffman(s, csym, ccnt, cn, 7, s.cl_len);
    png_codes(s.cl_len, 19, s.cl_code);
    int hclen = 4;
    for (int i = 0; i < 19; ++i)
        if (s.cl_len[png_cl_order(i)]) hclen = i + 1 > hclen ? i + 1 : hclen;
    s.hclen = hclen;
    int64_t hb = 3 + 5 + 5 + 4 + 3 * hclen;
    for (int i = 0; i < nr; ++i) hb += s.cl_len[s.rle_sym[i]] + png_cl_ext(s.rle_sym[i]);
    s.hdr_bits = hb;
}

// Thread 0: the dynamic block's header from bit 0.
__host__ __device__ __forceinline__ void png_header(PngSmem& s)
{
    PngBits w(s.out, 0);
    w.put(0u | (2u << 1), 3);                   // BFINAL 0, BTYPE 2
    w.put((uint32_t)(s.hlit - 257), 5);
    w.put(1u, 5);                               // HDIST - 1: two distance codes
    w.put((uint32_t)(s.hclen - 4), 4);
    for (int i = 0; i < s.hclen; ++i) w.put(s.cl_len[png_cl_order(i)], 3);
    for (int i = 0; i < s.n_rle; ++i) {
        const int sym = s.rle_sym[i];
        w.put(s.cl_code[sym], s.cl_len[sym]);
        if (png_cl_ext(sym)) w.put(s.rle_ext[i], png_cl_ext(sym));
    }
    w.flush();
}

enum {
    PNG_P_LOAD, PNG_P_BOUND, PNG_P_GROUP, PNG_P_TOP, PNG_P_COUNT, PNG_P_SORT, PNG_P_TREE, PNG_P_BITS, PNG_P_GROUP2, PNG_P_TOP2,
    PNG_P_EMIT, PNG_P_STORE, PNG_P_CRC0, PNG_P_FINAL = PNG_P_CRC0 + 10, PNG_SEG_PHASES
};

__host__ __device__ __forceinline__ void png_seg_phase(const PngArgs& a, PngSmem& s, int64_t c, int p, int t)
{
    const int64_t row0 = c * a.rows;
    const int nrows = (int)(a.H - row0 < a.rows ? a.H - row0 : a.rows);
    const int n = (int)(nrows * a.L);
    const int i0 = PNG_CHUNK * t, i1 = i0 + PNG_CHUNK < n ? i0 + PNG_CHUNK : n;
    const int g = t >> 5;
    if (p == PNG_P_LOAD) {
        const uint8_t* src = a.filt + row0 * a.L;
        for (int i = i0; i < i1; ++i) s.in[i] = src[i];
        for (int i = t; i < PNG_SLOT / 4; i += PNG_THREADS) s.out[i] = 0;
        if (t < PNG_LITLEN) s.hist[t] = t == 256;   // the end-of-block symbol
        if (t < 32) s.x2n[t] = png_x2n(t);
        if (t == 0) s.nused = 0;
    } else if (p == PNG_P_BOUND) {
        // first and last run start of the thread's bytes; its Adler-32 sums (s2 weights byte i by n - i)
        int fb = n, lb = -1;
        uint32_t s1 = 0; uint64_t s2 = 0;
        for (int i = i0; i < i1; ++i) {
            if (i == 0 || s.in[i] != s.in[i - 1]) { if (fb == n) fb = i; lb = i; }
            s1 += s.in[i]; s2 += (uint64_t)(n - i) * s.in[i];
        }
        s.fb[t] = fb; s.lb[t] = lb; s.s1[t] = s1; s.s2[t] = s2;
    } else if (p == PNG_P_GROUP) {
        if (t < 32) {
            int fb = n, lb = -1;
            uint64_t s1 = 0, s2 = 0;
            for (int j = 32 * t; j < 32 * t + 32; ++j) {
                if (s.fb[j] < fb) fb = s.fb[j];
                if (s.lb[j] > lb) lb = s.lb[j];
                s1 += s.s1[j]; s2 += s.s2[j];
            }
            s.gfb[t] = fb; s.glb[t] = lb;
            s.s1[32 * t] = (uint32_t)(s1 % PNG_ADLER_MOD); s.s2[32 * t] = s2 % PNG_ADLER_MOD;
        }
    } else if (p == PNG_P_TOP) {
        if (t == 0) {
            int m = -1;
            uint64_t s1 = 0, s2 = 0;
            for (int q = 0; q < 32; ++q) { s.gpre[q] = m; if (s.glb[q] > m) m = s.glb[q]; s1 += s.s1[32 * q]; s2 += s.s2[32 * q]; }
            m = n;
            for (int q = 31; q >= 0; --q) { s.gsuf[q] = m; if (s.gfb[q] < m) m = s.gfb[q]; }
            s.seg_s1 = (uint32_t)(s1 % PNG_ADLER_MOD); s.seg_s2 = (uint32_t)(s2 % PNG_ADLER_MOD);
        }
    } else if (p == PNG_P_COUNT) {
        // the start of the run holding byte i0 (the last run start before it) and the first run start at or after i1
        int rs = s.gpre[g], re = s.gsuf[g];
        for (int j = 32 * g; j < t; ++j) if (s.lb[j] > rs) rs = s.lb[j];
        for (int j = t + 1; j < 32 * g + 32; ++j) if (s.fb[j] < re) re = s.fb[j];
        s.rs0[t] = rs; s.re1[t] = re;
        png_walk<0>(s, n, t, 0);
    } else if (p == PNG_P_SORT) {
        if (t < PNG_LITLEN && s.hist[t]) {
            int r = 0;
            const uint32_t h = s.hist[t];
            for (int u = 0; u < PNG_LITLEN; ++u) r += s.hist[u] && (s.hist[u] < h || (s.hist[u] == h && u < t));
            s.sorted[r] = t;
            png_inc(&s.nused);
        }
    } else if (p == PNG_P_TREE) {
        if (t == 0) png_tree(s);
    } else if (p == PNG_P_BITS) {
        s.bits[t] = png_walk<1>(s, n, t, 0);
    } else if (p == PNG_P_GROUP2) {
        if (t < 32) {
            int64_t b = 0;
            for (int j = 32 * t; j < 32 * t + 32; ++j) b += s.bits[j];
            s.gbits[t] = b;
        }
    } else if (p == PNG_P_TOP2) {
        if (t == 0) {
            int64_t b = 0;
            for (int q = 0; q < 32; ++q) { s.gbpre[q] = b; b += s.gbits[q]; }
            s.tok_bits = b;
            // the dynamic block, the end-of-block code, then the sync flush: 3 bits, padding, 00 00 ff ff
            const int64_t dyn = (s.hdr_bits + b + s.len[256] + 3 + 7) / 8 + 4, stored = 5 + (int64_t)n;
            s.stored = dyn > stored;
            s.m = (int32_t)(s.stored ? stored : dyn);
        }
    } else if (p == PNG_P_EMIT) {
        if (s.stored) {
            uint8_t* o = (uint8_t*)s.out;
            for (int i = i0; i < i1; ++i) o[5 + i] = s.in[i];
            if (t == 0) { o[0] = 0; o[1] = (uint8_t)n; o[2] = (uint8_t)(n >> 8); o[3] = (uint8_t)~n; o[4] = (uint8_t)(~n >> 8); }
        } else {
            int64_t pos = s.hdr_bits + s.gbpre[g];
            for (int j = 32 * g; j < t; ++j) pos += s.bits[j];
            png_walk<2>(s, n, t, pos);
            if (t == 0) {
                png_header(s);
                PngBits w(s.out, s.hdr_bits + s.tok_bits);
                w.put(s.code[256], s.len[256]);
                w.flush();
                or_u32(s.out + ((s.m - 2) >> 2), 0xFFu << (8 * ((s.m - 2) & 3)));
                or_u32(s.out + ((s.m - 1) >> 2), 0xFFu << (8 * ((s.m - 1) & 3)));
            }
        }
    } else if (p == PNG_P_STORE) {
        const int m = s.m, words = (m + 3) >> 2;
        uint32_t* dst = (uint32_t*)(a.slots + c * PNG_SLOT);
        for (int i = t; i < words; i += PNG_THREADS) dst[i] = s.out[i];
        const auto [b0, b1] = thread_range<PNG_THREADS>(m, t);
        s.crc[t] = png_crc_bytes(0, (const uint8_t*)s.out + b0, b1 - b0);
    } else if (p < PNG_P_FINAL) {
        const int k = p - PNG_P_CRC0, m = s.m, q = (m + PNG_THREADS - 1) / PNG_THREADS;
        if ((t & ((2 << k) - 1)) == 0) {
            const int r = t + (1 << k);
            const int64_t lo = (int64_t)q * r < m ? (int64_t)q * r : m, hi = (int64_t)q * (r + (1 << k)) < m ? (int64_t)q * (r + (1 << k)) : m;
            s.crc[t] = png_crc_combine(s.x2n, s.crc[t], s.crc[r], hi - lo);
        }
    } else if (t == 0) {
        const uint8_t pre[6] = {'I', 'D', 'A', 'T', 0x78, 0x01};
        const uint32_t h = png_crc_bytes(0, pre, c == 0 ? 6 : 4);
        PngSeg& r = a.segs[c];
        r.n = (uint32_t)n; r.m = (uint32_t)s.m; r.crc = png_crc_combine(s.x2n, h, s.crc[0], s.m);
        r.s1 = s.seg_s1; r.s2 = s.seg_s2; r.pad = 0; r.off = 0;
    }
}

// ---------------------------------------------------------------- finish: one CTA
struct PngFinishSmem {
    uint64_t bytes[PNG_THREADS], n[PNG_THREADS]; uint32_t s1[PNG_THREADS], s2[PNG_THREADS];
    uint64_t gbytes[32], gpre[32];
};

__host__ __device__ __forceinline__ uint64_t png_chunk_bytes(const PngArgs& a, int64_t i)
{
    return 12 + a.segs[i].m + (i == 0 ? 2 : 0) + (i == a.S - 1 ? 6 : 0);
}

// Adler-32 sums of A || B from A's and B's (each from a = b = 0)
__host__ __device__ __forceinline__ void png_adler_cat(uint64_t& n, uint32_t& s1, uint32_t& s2, uint64_t nb, uint32_t s1b, uint32_t s2b)
{
    s2 = (uint32_t)((s2 + (uint64_t)s1 * (nb % PNG_ADLER_MOD) + s2b) % PNG_ADLER_MOD);
    s1 = (s1 + s1b) % PNG_ADLER_MOD;
    n += nb;
}

constexpr int64_t PNG_HEAD_BYTES = 8 + 25;      // signature, IHDR chunk

__host__ __device__ __forceinline__ void png_finish_phase(const PngArgs& a, PngFinishSmem& s, int64_t, int p, int t)
{
    const auto [j0, j1] = thread_range<PNG_THREADS>(a.S, t);
    const int g = t >> 5;
    if (p == 0) {
        uint64_t b = 0, n = 0; uint32_t s1 = 0, s2 = 0;
        for (int64_t i = j0; i < j1; ++i) { b += png_chunk_bytes(a, i); png_adler_cat(n, s1, s2, a.segs[i].n, a.segs[i].s1, a.segs[i].s2); }
        s.bytes[t] = b; s.n[t] = n; s.s1[t] = s1; s.s2[t] = s2;
    } else if (p == 1) {
        if (t < 32) {
            uint64_t b = 0, n = 0; uint32_t s1 = 0, s2 = 0;
            for (int j = 32 * t; j < 32 * t + 32; ++j) { b += s.bytes[j]; png_adler_cat(n, s1, s2, s.n[j], s.s1[j], s.s2[j]); }
            s.gbytes[t] = b; s.n[32 * t] = n; s.s1[32 * t] = s1; s.s2[32 * t] = s2;
        }
    } else if (p == 2) {
        if (t == 0) {
            uint64_t b = PNG_HEAD_BYTES, n = 0; uint32_t s1 = 0, s2 = 0;
            for (int k = 0; k < 32; ++k) { s.gpre[k] = b; b += s.gbytes[k]; png_adler_cat(n, s1, s2, s.n[32 * k], s.s1[32 * k], s.s2[32 * k]); }
            const uint32_t A = (1 + s1) % PNG_ADLER_MOD, B = (uint32_t)((n + s2) % PNG_ADLER_MOD);
            a.head->file_bytes = b + 12;
            a.head->adler = (B << 16) | A;
            const uint32_t ad = a.head->adler;
            const uint8_t tail[6] = {0x03, 0x00, (uint8_t)(ad >> 24), (uint8_t)(ad >> 16), (uint8_t)(ad >> 8), (uint8_t)ad};
            PngSeg& last = a.segs[a.S - 1];
            last.crc = png_crc_bytes(last.crc, tail, 6);
        }
    } else {
        uint64_t off = s.gpre[g];
        for (int j = 32 * g; j < t; ++j) off += s.bytes[j];
        for (int64_t i = j0; i < j1; ++i) { a.segs[i].off = off; off += png_chunk_bytes(a, i); }
    }
}
constexpr int PNG_FINISH_PHASES = 4;

// ---------------------------------------------------------------- write: one CTA per chunk, the last for the rest
__host__ __device__ __forceinline__ void png_be32(uint8_t* p, uint32_t v)
{
    p[0] = (uint8_t)(v >> 24); p[1] = (uint8_t)(v >> 16); p[2] = (uint8_t)(v >> 8); p[3] = (uint8_t)v;
}

__host__ __device__ __forceinline__ void png_write_block(const PngArgs& a, int64_t c, int t)
{
    if (c < a.S) {
        const PngSeg& r = a.segs[c];
        uint8_t* o = a.out + r.off;
        const int pre = c == 0 ? 2 : 0;
        const uint32_t data = r.m + pre + (c == a.S - 1 ? 6 : 0);
        const uint8_t* src = a.slots + c * PNG_SLOT;
        for (int64_t i = t; i < r.m; i += PNG_THREADS) o[8 + pre + i] = src[i];
        if (t == 0) {
            png_be32(o, data);
            o[4] = 'I'; o[5] = 'D'; o[6] = 'A'; o[7] = 'T';
            if (pre) { o[8] = 0x78; o[9] = 0x01; }
            png_be32(o + 8 + data, r.crc);
        }
        return;
    }
    if (t != 0) return;
    uint8_t* o = a.out;
    const uint8_t sig[8] = {0x89, 'P', 'N', 'G', 0x0D, 0x0A, 0x1A, 0x0A};
    for (int i = 0; i < 8; ++i) o[i] = sig[i];
    uint8_t* h = o + 8;
    png_be32(h, 13);
    h[4] = 'I'; h[5] = 'H'; h[6] = 'D'; h[7] = 'R';
    png_be32(h + 8, (uint32_t)a.W); png_be32(h + 12, (uint32_t)a.H);
    h[16] = 8; h[17] = 2; h[18] = 0; h[19] = 0; h[20] = 0;        // 8-bit RGB, deflate, adaptive filtering, no interlace
    png_be32(h + 21, png_crc_bytes(0, h + 4, 17));
    const PngSeg& last = a.segs[a.S - 1];
    uint8_t* tl = o + last.off + 8 + (a.S == 1 ? 2 : 0) + last.m;
    tl[0] = 0x03; tl[1] = 0x00;                 // the final block: fixed Huffman, end of block
    png_be32(tl + 2, a.head->adler);
    uint8_t* e = o + a.head->file_bytes - 12;
    const uint8_t iend[12] = {0, 0, 0, 0, 'I', 'E', 'N', 'D', 0xAE, 0x42, 0x60, 0x82};
    for (int i = 0; i < 12; ++i) e[i] = iend[i];
}

// ---------------------------------------------------------------- kernels
__global__ void __launch_bounds__(PNG_THREADS) png_write_kernel(const PngArgs a)
{
    png_write_block(a, blockIdx.x, threadIdx.x);
}

}  // namespace perf

using namespace perf;

static bool png_shape_ok(int H, int W) { return H >= 1 && W >= 1 && W <= PNG_MAX_W; }

struct PngLayout { uint64_t filt, slots, segs, head, total; int32_t rows; int64_t S; };

static PngLayout png_layout(int H, int W)
{
    PngLayout l;
    const int64_t L = 1 + 3 * (int64_t)W;
    l.rows = (int32_t)(PNG_SEG_MAX / L);
    l.S = (H + (int64_t)l.rows - 1) / l.rows;
    auto up = [](uint64_t v) { return (v + 255) & ~(uint64_t)255; };
    l.filt = 0;
    l.slots = up((uint64_t)H * L);
    l.segs = l.slots + (uint64_t)l.S * PNG_SLOT;
    l.head = up(l.segs + (uint64_t)l.S * sizeof(PngSeg));
    l.total = l.head + 256;
    return l;
}

static int png_args(PngArgs& a, const uint8_t* image, int H, int W, void* ws, uint64_t ws_bytes)
{
    PERF_CHECK_ARG(png_shape_ok(H, W), "png image %d x %d: needs 1 <= H and 1 <= W <= %d", H, W, PNG_MAX_W);
    PERF_CHECK_ARG(ws && (uintptr_t)ws % 16 == 0, "workspace NULL or not 16-byte aligned");
    const PngLayout l = png_layout(H, W);
    PERF_CHECK_ARG(ws_bytes >= l.total, "workspace of %llu bytes, needs %llu", (unsigned long long)ws_bytes, (unsigned long long)l.total);
    PERF_CHECK_ARG(l.S < (1ll << 31), "%lld segments", (long long)l.S);
    memset(&a, 0, sizeof(a));
    uint8_t* w = (uint8_t*)ws;
    a.image = image; a.filt = w + l.filt; a.slots = w + l.slots; a.segs = (PngSeg*)(w + l.segs); a.head = (PngHead*)(w + l.head);
    a.H = H; a.W = W; a.rows = l.rows; a.L = 1 + 3 * (int64_t)W; a.S = l.S;
    return PERF_OK;
}

extern "C" {
#pragma GCC visibility push(default)

uint64_t perf_png_workspace_bytes(int H, int W)
{
    return png_shape_ok(H, W) ? png_layout(H, W).total : 0;
}

uint64_t perf_png_max_bytes(int H, int W)
{
    if (!png_shape_ok(H, W)) return 0;
    const PngLayout l = png_layout(H, W);
    return (uint64_t)PNG_HEAD_BYTES + (uint64_t)l.S * 17 + (uint64_t)H * (1 + 3 * (uint64_t)W) + 2 + 6 + 12;
}

int perf_png_compress(const uint8_t* d_image, int H, int W, void* d_workspace, uint64_t workspace_bytes, void* stream)
{
    PngArgs a;
    int rc = png_args(a, d_image, H, W, d_workspace, workspace_bytes); if (rc) return rc;
    PERF_CHECK_ARG(d_image, "NULL image");
    const cudaStream_t st = (cudaStream_t)stream;
    rc = run_cta_phases<PngArgs, PngFilterSmem, PNG_FILTER_THREADS, PNG_FILTER_PHASES, png_filter_phase>(a, H, st); if (rc) return rc;
    rc = run_cta_phases<PngArgs, PngSmem, PNG_THREADS, PNG_SEG_PHASES, png_seg_phase>(a, a.S, st); if (rc) return rc;
    return run_cta_phases<PngArgs, PngFinishSmem, PNG_THREADS, PNG_FINISH_PHASES, png_finish_phase>(a, 1, st);
}

int perf_png_write(const void* d_workspace, uint64_t workspace_bytes, int H, int W, uint8_t* d_out, uint64_t out_bytes,
                   uint64_t* d_file_bytes, void* stream)
{
    PngArgs a;
    int rc = png_args(a, nullptr, H, W, (void*)d_workspace, workspace_bytes); if (rc) return rc;
    PERF_CHECK_ARG(d_out && d_file_bytes, "NULL pointer");
    PERF_CHECK_ARG(out_bytes >= perf_png_max_bytes(H, W), "output of %llu bytes, needs %llu", (unsigned long long)out_bytes,
                   (unsigned long long)perf_png_max_bytes(H, W));
    a.out = d_out;
#ifdef PERF_HOST_HARNESS
    (void)stream;
    for (int64_t c = 0; c <= a.S; ++c)
        for (int t = 0; t < PNG_THREADS; ++t) png_write_block(a, c, t);
    *d_file_bytes = a.head->file_bytes;
#else
    png_write_kernel<<<(unsigned)(a.S + 1), PNG_THREADS, 0, (cudaStream_t)stream>>>(a);
    PERF_LAUNCH_CHECK();
    PERF_CUDA(cudaMemcpyAsync(d_file_bytes, &a.head->file_bytes, sizeof(uint64_t), cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
#endif
    return PERF_OK;
}

#pragma GCC visibility pop
}
