// h264.cu -- intra-only H.264 encoder (8-bit RGB frames in, Constrained Baseline IDR access units out) with all of the coding
// on the GPU.  Every frame is one IDR picture of one CAVLC slice; every macroblock is Intra 16x16, Intra 4x4 or I_PCM.  Launches in
// perf_h264_encode:
//   mb       (one thread per macroblock, one launch per wavefront t = x + 2 y, every frame of the batch in each launch):
//            colour conversion, the Intra 16x16, Intra 4x4 and chroma mode search, transform, quantisation, reconstruction into the Y/Cb/Cr
//            workspace, the quantised levels, every 4x4 block's total_coeff and the macroblock's exact CAVLC bit count (its left
//            and top neighbours finished in earlier launches, so nC is known); a macroblock over the A.3.1 limit becomes I_PCM;
//   scan     (one CTA per frame): the bit offset of every macroblock in the slice (I_PCM's byte alignment depends on the
//            position, so each thread's run of macroblocks is scanned for all 8 starting bit phases), the frame's slot zeroed;
//   emit     (one thread per macroblock): the slice header, the macroblock's codes and the RBSP trailing bits ORed into the
//            frame's slot, word by word;
//   nal      (one CTA per frame): emulation prevention (each thread's run of bytes is scanned for the 3 zero-run states it can
//            start in), the access unit as a 4-byte big-endian length and the NAL unit into the frame's staging slot;
//   finish   (one CTA): every access unit's offset in the output and the total.
// perf_h264_write (one CTA per frame) copies the access units out.  Integer arithmetic only; the only atomics are integer
// ORs, so the bytes do not depend on execution order, and the host build of tests/h264_harness.py (-DPERF_HOST_HARNESS: each
// thread's or CTA's phases over host arrays in a serial loop) agrees bit for bit.  Rule: perfb200.h (perf_h264_*).
#include "common.cuh"

namespace perf {

constexpr int H264_MAX_MBS = 139264;            // MaxFS of level 6.2 (Table A-1)
constexpr int H264_MB_MAX_BITS = 5934;          // A.3.1: 128 + RawMbBits 189 / 100, RawMbBits = 384 * 8
// Macroblocks coded in more bits than this become I_PCM.  The A.3.1 limit; test builds of the host harness lower it, because
// with Intra 4x4 no ordinary content reaches it and the I_PCM syntax would go unchecked.  The workspace is always sized for
// H264_MB_MAX_BITS.
#ifndef PERF_H264_PCM_ABOVE_BITS
#define PERF_H264_PCM_ABOVE_BITS H264_MB_MAX_BITS
#endif
constexpr int H264_PCM_BITS = 3072;             // 384 samples; plus ue(25) (9 bits) and the byte alignment before them
constexpr int H264_SLICE_MAX_BITS = 64;         // the slice header is at most 32 bits
constexpr int H264_MB_THREADS = 64;
constexpr int H264_FRAME_THREADS = 256;
constexpr int H264_LEVELS = 384;                // per macroblock: luma DC 16, luma AC 16 x 15, chroma DC 2 x 4, chroma AC 8 x 15

struct H264Tables {
    uint8_t ct_len[4][17][4], ct_code[4][17][4];    // coeff_token (Table 9-5): nC 0-1, 2-3, 4-7, >= 8; [TotalCoeff][T1s]
    uint8_t cdc_len[5][4], cdc_code[5][4];          // coeff_token, nC = -1 (chroma DC)
    uint8_t tz_len[15][16], tz_code[15][16];        // total_zeros, 4x4 blocks (Tables 9-7, 9-8); [TotalCoeff - 1][total_zeros]
    uint8_t ctz_len[3][4], ctz_code[3][4];          // total_zeros, chroma DC (Table 9-9a)
    uint8_t rb_len[7][15], rb_code[7][15];          // run_before (Table 9-10); [min(zerosLeft, 7) - 1][run_before]
    uint8_t cbp_code[48];                           // coded_block_pattern -> codeNum of me(v), Intra_4x4 (Table 9-4)
};

// Per macroblock: mode 0-3 the Intra 16x16 prediction mode (vertical, horizontal, DC, plane), 4 I_PCM, 5 Intra 4x4; cmode the
// chroma mode (DC, horizontal, vertical, plane); cbp_l 15 or 0 (Intra 16x16) or one bit per 8x8 block (Intra 4x4); m4 the
// Intra4x4PredMode of the 4x4 blocks in raster order (x + 4 y), 2 (DC) in other macroblocks, as the most probable mode of their
// neighbours sees them; tc the total_coeff of the 4x4 blocks as nC sees them: luma in raster order, then Cb and Cr in raster
// order (16 for every block of an I_PCM macroblock).  The first 20 bytes are what perf_h264_mb_modes copies out.
struct H264Mb { uint8_t mode, cmode, cbp_l, cbp_c; uint8_t m4[16]; uint8_t tc[24]; };
struct H264Frame { uint32_t bits, pad; uint64_t au, off; };

struct H264Args {
    const uint8_t* rgb; uint8_t* rec; H264Mb* mb; int16_t* lev; uint32_t* mbits; uint32_t* moff; H264Frame* fr;
    uint8_t* slots; uint8_t* nals; uint64_t* total; uint8_t* out;
    uint64_t out_bytes;
    int32_t N, H, W, MX, MY, qp, t;             // t: the anti-diagonal of the mb launch
    int64_t M;                                  // macroblocks per frame
    uint64_t plane, slot, nal;                  // workspace bytes per frame: reconstruction, unescaped slice data, staging
    H264Tables tab;
};

__host__ __device__ __forceinline__ int h264_clip(int v) { return v < 0 ? 0 : v > 255 ? 255 : v; }

// Exp-Golomb codes (9.1) into a bit sink (common.cuh: BitCount, MsbBits)
template <class S> __host__ __device__ __forceinline__ void h264_ue(S& s, uint32_t v) { s.put(v + 1, 2 * bit_width(v + 1) - 1); }
template <class S> __host__ __device__ __forceinline__ void h264_se(S& s, int v) { h264_ue(s, v > 0 ? 2 * v - 1 : -2 * v); }

// Raster index (x + 4 y) of 4x4 zigzag position k, and of luma4x4BlkIdx b's block in the macroblock
__host__ __device__ __forceinline__ int h264_zz(int k) { return (uint8_t)"\x00\x01\x04\x08\x05\x02\x03\x06\x09\x0c\x0d\x0a\x07\x0b\x0e\x0f"[k]; }
__host__ __device__ __forceinline__ int h264_blk(int b) { return (b & 1) + ((b >> 1) & 1) * 4 + ((b >> 2) & 1) * 2 + ((b >> 3) & 1) * 8; }
__host__ __device__ __forceinline__ int h264_blkidx(int r) { return (r & 1) + ((r >> 2) & 1) * 2 + ((r >> 1) & 1) * 4 + ((r >> 3) & 1) * 8; }

// Table 8-15 (chroma_qp_index_offset 0), the quantiser multipliers and LevelScale by qP % 6 and position class (0: both
// coordinates even, 1: both odd, 2: mixed), and the mode-decision lambda round(0.85 2^((QP - 12) / 6)), at least 1.
__host__ __device__ __forceinline__ int h264_qpc(int qp)
{
    return qp < 30 ? qp : (uint8_t)"\x1d\x1e\x1f\x20\x20\x21\x22\x22\x23\x23\x24\x24\x25\x25\x25\x26\x26\x26\x27\x27\x27\x27"[qp - 30];
}
__host__ __device__ __forceinline__ int h264_mf(int m, int c)
{
    const int t[6][3] = {{13107, 5243, 8066}, {11916, 4660, 7490}, {10082, 4194, 6554}, {9362, 3647, 5825}, {8192, 3355, 5243}, {7282, 2893, 4559}};
    return t[m][c];
}
__host__ __device__ __forceinline__ int h264_ls(int m, int c)
{
    const int t[6][3] = {{10, 16, 13}, {11, 18, 14}, {13, 20, 16}, {14, 23, 18}, {16, 25, 20}, {18, 29, 23}};
    return t[m][c];
}
__host__ __device__ __forceinline__ int h264_cls(int i) { const int x = i & 1, y = (i >> 2) & 1; return x == y ? x : 2; }
__host__ __device__ __forceinline__ int h264_lambda(int qp)
{
    return (uint8_t)"\x01\x01\x01\x01\x01\x01\x01\x01\x01\x01\x01\x01\x01\x01\x01\x01\x01\x02\x02\x02\x02\x02\x03\x03\x03\x04"
                    "\x04\x05\x05\x06\x07\x08\x09\x0a\x0b\x0c\x0e\x0f\x11\x13\x16\x18\x1b\x1f\x22\x26\x2b\x30\x36\x3d\x45\x4d"[qp];
}

// ---------------------------------------------------------------- transforms (8.5.12, and their forward counterparts)
__host__ __device__ __forceinline__ void h264_fdct(int d[16])
{
    for (int p = 0; p < 2; ++p)
        for (int i = 0; i < 4; ++i) {
            const int s = p ? 4 : 1, o = p ? i : 4 * i;         // rows, then columns
            const int a = d[o], b = d[o + s], c = d[o + 2 * s], e = d[o + 3 * s];
            const int s03 = a + e, d03 = a - e, s12 = b + c, d12 = b - c;
            d[o] = s03 + s12; d[o + s] = 2 * d03 + d12; d[o + 2 * s] = s03 - s12; d[o + 3 * s] = d03 - 2 * d12;
        }
}
__host__ __device__ __forceinline__ void h264_idct(int d[16])
{
    for (int p = 0; p < 2; ++p)
        for (int i = 0; i < 4; ++i) {
            const int s = p ? 4 : 1, o = p ? i : 4 * i;
            const int a = d[o], b = d[o + s], c = d[o + 2 * s], e = d[o + 3 * s];
            const int e0 = a + c, e1 = a - c, e2 = (b >> 1) - e, e3 = b + (e >> 1);
            d[o] = e0 + e3; d[o + s] = e1 + e2; d[o + 2 * s] = e1 - e2; d[o + 3 * s] = e0 - e3;
        }
    for (int i = 0; i < 16; ++i) d[i] = (d[i] + 32) >> 6;
}
__host__ __device__ __forceinline__ void h264_hadamard(int d[16])
{
    for (int p = 0; p < 2; ++p)
        for (int i = 0; i < 4; ++i) {
            const int s = p ? 4 : 1, o = p ? i : 4 * i;
            const int a = d[o], b = d[o + s], c = d[o + 2 * s], e = d[o + 3 * s];
            d[o] = a + b + c + e; d[o + s] = a + b - c - e; d[o + 2 * s] = a - b - c + e; d[o + 3 * s] = a - b + c - e;
        }
}
// 4x4 SATD: the Hadamard transform of the difference, sum of magnitudes / 2
__host__ __device__ __forceinline__ int h264_satd(const uint8_t* src, int ss, const uint8_t* pred, int ps)
{
    int d[16];
    for (int j = 0; j < 4; ++j)
        for (int i = 0; i < 4; ++i) d[4 * j + i] = (int)src[j * ss + i] - (int)pred[j * ps + i];
    h264_hadamard(d);
    int s = 0;
    for (int i = 0; i < 16; ++i) s += d[i] < 0 ? -d[i] : d[i];
    return s >> 1;
}
__host__ __device__ __forceinline__ int h264_quant(int v, int mf, int f, int sh)
{
    return v < 0 ? -((-v * mf + f) >> sh) : (v * mf + f) >> sh;
}

// ---------------------------------------------------------------- intra prediction (8.3.3, 8.3.4)
// n x n block (16 luma, 8 chroma) from the top row t[0..n-1], the left column l[0..n-1] and the corner c; ut / ul: top / left
// available.  Luma modes 0 V, 1 H, 2 DC, 3 plane; chroma modes 0 DC (per 4x4 block), 1 H, 2 V, 3 plane.
__host__ __device__ __forceinline__ void h264_pred(uint8_t* p, int n, bool chroma, int mode, const uint8_t* t, const uint8_t* l, int c,
                                                   bool ut, bool ul)
{
    const int m = chroma ? (mode == 0 ? 2 : mode == 2 ? 0 : mode) : mode;   // chroma renumbered to the luma order
    if (m == 0) { for (int j = 0; j < n; ++j) for (int i = 0; i < n; ++i) p[n * j + i] = t[i]; return; }
    if (m == 1) { for (int j = 0; j < n; ++j) for (int i = 0; i < n; ++i) p[n * j + i] = l[j]; return; }
    if (m == 3) {
        const int h2 = n / 2;
        int Hs = 0, Vs = 0;
        for (int k = 0; k < h2; ++k) {
            Hs += (k + 1) * (t[h2 + k] - (h2 - 2 - k >= 0 ? t[h2 - 2 - k] : c));
            Vs += (k + 1) * (l[h2 + k] - (h2 - 2 - k >= 0 ? l[h2 - 2 - k] : c));
        }
        const int A = 16 * (l[n - 1] + t[n - 1]);
        const int B = chroma ? (34 * Hs + 32) >> 6 : (5 * Hs + 32) >> 6, C = chroma ? (34 * Vs + 32) >> 6 : (5 * Vs + 32) >> 6;
        for (int j = 0; j < n; ++j)
            for (int i = 0; i < n; ++i) p[n * j + i] = (uint8_t)h264_clip((A + B * (i - (h2 - 1)) + C * (j - (h2 - 1)) + 16) >> 5);
        return;
    }
    if (!chroma) {
        int s = 0, v;
        for (int k = 0; k < 16; ++k) s += (ut ? t[k] : 0) + (ul ? l[k] : 0);
        v = ut && ul ? (s + 16) >> 5 : ut || ul ? (s + 8) >> 4 : 128;
        for (int k = 0; k < 256; ++k) p[k] = (uint8_t)v;
        return;
    }
    for (int by = 0; by < 2; ++by)
        for (int bx = 0; bx < 2; ++bx) {
            int st = 0, sl = 0;
            for (int k = 0; k < 4; ++k) { st += t[4 * bx + k]; sl += l[4 * by + k]; }
            int v;
            if (bx == by) v = ut && ul ? (st + sl + 4) >> 3 : ul ? (sl + 2) >> 2 : ut ? (st + 2) >> 2 : 128;
            else if (bx) v = ut ? (st + 2) >> 2 : ul ? (sl + 2) >> 2 : 128;
            else v = ul ? (sl + 2) >> 2 : ut ? (st + 2) >> 2 : 128;
            for (int j = 0; j < 4; ++j)
                for (int i = 0; i < 4; ++i) p[8 * (4 * by + j) + 4 * bx + i] = (uint8_t)v;
        }
}

// Intra 4x4 (8.3.1.2) into p (raster) from e[13]: e[3 - y] = p[-1, y] (y = -1 .. 3), e[5 + x] = p[x, -1] (x = -1 .. 7; the
// caller repeats p[3, -1] when the top-right samples are not available).  Modes 0 vertical, 1 horizontal, 2 DC, 3 diagonal
// down-left, 4 diagonal down-right, 5 vertical-right, 6 horizontal-down, 7 vertical-left, 8 horizontal-up; ut / ul: top / left.
__host__ __device__ __forceinline__ void h264_pred4(uint8_t* p, int md, const int* e, bool ut, bool ul)
{
    auto T = [&](int x) { return e[5 + x]; };
    auto L = [&](int y) { return e[3 - y]; };
    for (int y = 0; y < 4; ++y)
        for (int x = 0; x < 4; ++x) {
            int v, z;
            switch (md) {
            case 0: v = T(x); break;
            case 1: v = L(y); break;
            case 2: {
                const int st = T(0) + T(1) + T(2) + T(3), sl = L(0) + L(1) + L(2) + L(3);
                v = ut && ul ? (st + sl + 4) >> 3 : ul ? (sl + 2) >> 2 : ut ? (st + 2) >> 2 : 128;
                break;
            }
            case 3: v = x == 3 && y == 3 ? (T(6) + 3 * T(7) + 2) >> 2 : (T(x + y) + 2 * T(x + y + 1) + T(x + y + 2) + 2) >> 2; break;
            case 4:
                v = x > y ? (T(x - y - 2) + 2 * T(x - y - 1) + T(x - y) + 2) >> 2
                  : x < y ? (L(y - x - 2) + 2 * L(y - x - 1) + L(y - x) + 2) >> 2 : (T(0) + 2 * T(-1) + L(0) + 2) >> 2;
                break;
            case 5:
                z = 2 * x - y;
                v = z >= 0 && !(z & 1) ? (T(x - (y >> 1) - 1) + T(x - (y >> 1)) + 1) >> 1
                  : z >= 0 ? (T(x - (y >> 1) - 2) + 2 * T(x - (y >> 1) - 1) + T(x - (y >> 1)) + 2) >> 2
                  : z == -1 ? (L(0) + 2 * L(-1) + T(0) + 2) >> 2 : (L(y - 1) + 2 * L(y - 2) + L(y - 3) + 2) >> 2;
                break;
            case 6:
                z = 2 * y - x;
                v = z >= 0 && !(z & 1) ? (L(y - (x >> 1) - 1) + L(y - (x >> 1)) + 1) >> 1
                  : z >= 0 ? (L(y - (x >> 1) - 2) + 2 * L(y - (x >> 1) - 1) + L(y - (x >> 1)) + 2) >> 2
                  : z == -1 ? (L(0) + 2 * L(-1) + T(0) + 2) >> 2 : (T(x - 1) + 2 * T(x - 2) + T(x - 3) + 2) >> 2;
                break;
            case 7:
                v = !(y & 1) ? (T(x + (y >> 1)) + T(x + (y >> 1) + 1) + 1) >> 1
                             : (T(x + (y >> 1)) + 2 * T(x + (y >> 1) + 1) + T(x + (y >> 1) + 2) + 2) >> 2;
                break;
            default:
                z = x + 2 * y;
                v = z > 5 ? L(3) : z == 5 ? (L(2) + 3 * L(3) + 2) >> 2
                  : !(z & 1) ? (L(y + (x >> 1)) + L(y + (x >> 1) + 1) + 1) >> 1
                  : (L(y + (x >> 1)) + 2 * L(y + (x >> 1) + 1) + L(y + (x >> 1) + 2) + 2) >> 2;
            }
            p[4 * y + x] = (uint8_t)v;
        }
}

// predIntra4x4PredMode (8.3.1.1) of raster block r: the smaller of the left and top blocks' modes (2 for a neighbour that is
// not Intra 4x4), 2 when either is outside the picture
__host__ __device__ __forceinline__ int h264_mpm(const H264Mb& m, const H264Mb* ml, const H264Mb* mt, int r)
{
    const int x = r & 3, y = r >> 2;
    const int A = x ? m.m4[r - 1] : ml ? ml->m4[r + 3] : -1, B = y ? m.m4[r - 4] : mt ? mt->m4[r + 12] : -1;
    return A < 0 || B < 0 ? 2 : A < B ? A : B;
}

// ---------------------------------------------------------------- CAVLC residual_block (9.2)
// c: the block's levels in coding order, n = maxNumCoeff (16, 15 or 4); nC < 0 for chroma DC.  Returns false when a level
// needs level_prefix > 15, which Baseline streams may not use.
template <class S>
__host__ __device__ __forceinline__ bool h264_cavlc(S& s, const H264Tables& tb, const int16_t* c, int n, int nC)
{
    int lv[16], idx[16], tc = 0;
    for (int i = n - 1; i >= 0; --i)
        if (c[i]) { lv[tc] = c[i]; idx[tc] = i; ++tc; }
    int t1 = 0;
    while (t1 < tc && t1 < 3 && (lv[t1] == 1 || lv[t1] == -1)) ++t1;
    if (nC < 0) s.put(tb.cdc_code[tc][t1], tb.cdc_len[tc][t1]);
    else {
        const int k = nC < 2 ? 0 : nC < 4 ? 1 : nC < 8 ? 2 : 3;
        s.put(tb.ct_code[k][tc][t1], tb.ct_len[k][tc][t1]);
    }
    if (tc == 0) return true;
    for (int k = 0; k < t1; ++k) s.put(lv[k] < 0, 1);
    int sl = tc > 10 && t1 < 3 ? 1 : 0;
    for (int k = t1; k < tc; ++k) {
        const int v = lv[k];
        int code = v > 0 ? 2 * v - 2 : -2 * v - 1;
        if (k == t1 && t1 < 3) code -= 2;
        if (sl == 0) {
            if (code < 14) s.put(1, code + 1);
            else if (code < 30) { s.put(1, 15); s.put(code - 14, 4); }
            else { if (code - 30 >= 4096) return false; s.put(1, 16); s.put(code - 30, 12); }
        } else {
            if (code < (15 << sl)) { s.put(1, (code >> sl) + 1); s.put(code & ((1 << sl) - 1), sl); }
            else { if (code - (15 << sl) >= 4096) return false; s.put(1, 16); s.put(code - (15 << sl), 12); }
        }
        if (sl == 0) sl = 1;
        if ((v < 0 ? -v : v) > (3 << (sl - 1)) && sl < 6) ++sl;
    }
    int zl = idx[0] + 1 - tc;
    if (tc < n) {
        if (n == 4) s.put(tb.ctz_code[tc - 1][zl], tb.ctz_len[tc - 1][zl]);
        else s.put(tb.tz_code[tc - 1][zl], tb.tz_len[tc - 1][zl]);
    }
    for (int k = 0; k < tc - 1 && zl > 0; ++k) {
        const int r = idx[k] - idx[k + 1] - 1, z = (zl < 7 ? zl : 7) - 1;
        s.put(tb.rb_code[z][r], tb.rb_len[z][r]);
        zl -= r;
    }
    return true;
}

__host__ __device__ __forceinline__ int h264_nc(int a, int b)
{
    return a >= 0 && b >= 0 ? (a + b + 1) >> 1 : a >= 0 ? a : b >= 0 ? b : 0;
}

// The macroblock_layer of a non-PCM macroblock (7.3.5): mb_type; Intra 4x4: the 16 prediction modes (prev_intra4x4_pred_mode_flag,
// rem_intra4x4_pred_mode), intra_chroma_pred_mode, coded_block_pattern, mb_qp_delta 0 when it is not 0; Intra 16x16:
// intra_chroma_pred_mode, mb_qp_delta 0; then the residual.
// m: this macroblock, ml / mt: its left / top neighbours (null when outside the picture).  false: a level is not codable.
template <class S>
__host__ __device__ __forceinline__ bool h264_mb_syntax(S& s, const H264Tables& tb, const H264Mb& m, const H264Mb* ml, const H264Mb* mt,
                                                        const int16_t* lev)
{
    bool ok = true;
    auto luma_nc = [&](int r) {
        const int x = r & 3, y = r >> 2;
        const int a = x ? m.tc[r - 1] : ml ? ml->tc[r + 3] : -1, b = y ? m.tc[r - 4] : mt ? mt->tc[r + 12] : -1;
        return h264_nc(a, b);
    };
    if (m.mode == 5) {
        s.put(1, 1);                                // ue(0): I_NxN
        for (int b = 0; b < 16; ++b) {
            const int r = h264_blk(b), pm = h264_mpm(m, ml, mt, r), md = m.m4[r];
            if (md == pm) s.put(1, 1);
            else s.put(md < pm ? md : md - 1, 4);   // flag 0, then 3 bits
        }
        h264_ue(s, m.cmode);
        h264_ue(s, tb.cbp_code[m.cbp_l | m.cbp_c << 4]);
        if (m.cbp_l || m.cbp_c) s.put(1, 1);
        for (int b = 0; b < 16; ++b)
            if ((m.cbp_l >> (b >> 2)) & 1) ok &= h264_cavlc(s, tb, lev + 16 * b, 16, luma_nc(h264_blk(b)));
    } else {
        h264_ue(s, 1 + m.mode + 4 * m.cbp_c + (m.cbp_l ? 12 : 0));
        h264_ue(s, m.cmode);
        s.put(1, 1);
        ok &= h264_cavlc(s, tb, lev, 16, luma_nc(0));
        if (m.cbp_l)
            for (int b = 0; b < 16; ++b) ok &= h264_cavlc(s, tb, lev + 16 + 15 * b, 15, luma_nc(h264_blk(b)));
    }
    if (m.cbp_c) {
        ok &= h264_cavlc(s, tb, lev + 256, 4, -1);
        ok &= h264_cavlc(s, tb, lev + 260, 4, -1);
    }
    if (m.cbp_c == 2)
        for (int p = 0; p < 2; ++p)
            for (int b = 0; b < 4; ++b) {
                const int o = 16 + 4 * p, x = b & 1, y = b >> 1;
                const int a = x ? m.tc[o + b - 1] : ml ? ml->tc[o + b + 1] : -1, c = y ? m.tc[o + b - 2] : mt ? mt->tc[o + b + 2] : -1;
                ok &= h264_cavlc(s, tb, lev + 264 + 60 * p + 15 * b, 15, h264_nc(a, c));
            }
    return ok;
}

// slice_header (7.3.3) of frame f: I slice, frame_num 0, idr_pic_id f & 1, slice_qp_delta qp - 26, deblocking off
template <class S> __host__ __device__ __forceinline__ void h264_slice_header(S& s, int f, int qp)
{
    h264_ue(s, 0); h264_ue(s, 7); h264_ue(s, 0);
    s.put(0, 4);
    h264_ue(s, f & 1);
    s.put(0, 2);
    h264_se(s, qp - 26);
    h264_ue(s, 1);
}

// ---------------------------------------------------------------- mb: one thread per macroblock of anti-diagonal t
__host__ __device__ __forceinline__ uint8_t* h264_plane(const H264Args& a, int64_t f, int c)
{
    const int64_t PW = 16 * (int64_t)a.MX, PH = 16 * (int64_t)a.MY;
    return a.rec + f * a.plane + (c == 0 ? 0 : PW * PH + (c - 1) * (PW / 2) * (PH / 2));
}

__host__ __device__ __forceinline__ void h264_mb(const H264Args& a, const H264Tables& tb, int64_t f, int mx, int my)
{
    const int64_t mi = f * a.M + (int64_t)my * a.MX + mx;
    const int PW = 16 * a.MX;
    int16_t* lev = a.lev + mi * H264_LEVELS;
    uint8_t src[384];                           // Y 16 x 16, Cb 8 x 8, Cr 8 x 8
    for (int j = 0; j < 16; ++j)
        for (int i = 0; i < 16; ++i) {
            const int x = 16 * mx + i < a.W ? 16 * mx + i : a.W - 1, y = 16 * my + j < a.H ? 16 * my + j : a.H - 1;
            const uint8_t* p = a.rgb + ((f * a.H + y) * a.W + x) * 3;
            src[16 * j + i] = (uint8_t)(((66 * p[0] + 129 * p[1] + 25 * p[2] + 128) >> 8) + 16);
        }
    for (int j = 0; j < 8; ++j)
        for (int i = 0; i < 8; ++i) {
            int cb = 0, cr = 0;
            for (int k = 0; k < 4; ++k) {
                const int xx = 16 * mx + 2 * i + (k & 1), yy = 16 * my + 2 * j + (k >> 1);
                const int x = xx < a.W ? xx : a.W - 1, y = yy < a.H ? yy : a.H - 1;
                const uint8_t* p = a.rgb + ((f * a.H + y) * a.W + x) * 3;
                cb += ((-38 * p[0] - 74 * p[1] + 112 * p[2] + 128) >> 8) + 128;
                cr += ((112 * p[0] - 94 * p[1] - 18 * p[2] + 128) >> 8) + 128;
            }
            src[256 + 8 * j + i] = (uint8_t)((cb + 2) >> 2);
            src[320 + 8 * j + i] = (uint8_t)((cr + 2) >> 2);
        }
    const bool ut = my > 0, ul = mx > 0;
    const int lam = h264_lambda(a.qp), qp = a.qp, qpc = h264_qpc(a.qp);
    uint8_t rec[384], pred[256], best[256];
    H264Mb m;
    for (int k = 0; k < 16; ++k) m.m4[k] = 2;
    const H264Mb* ml = ul ? a.mb + mi - 1 : nullptr;
    const H264Mb* mt = ut ? a.mb + mi - a.MX : nullptr;
    // ---- luma: the Intra 16x16 mode of least SATD + lambda bits(mb_type), against Intra 4x4 (per block the mode of least
    // SATD + lambda bits(mode), 1 for the most probable mode, else 4; plus lambda for mb_type)
    {
        const uint8_t* Y = h264_plane(a, f, 0) + (int64_t)16 * my * PW + 16 * mx;
        uint8_t t[16], l[16];
        for (int k = 0; k < 16; ++k) { t[k] = ut ? Y[k - PW] : 0; l[k] = ul ? Y[(int64_t)k * PW - 1] : 0; }
        const int c = ut && ul ? Y[-PW - 1] : 0;
        int bc = 0x7fffffff;
        m.mode = 2;
        for (int md = 0; md < 4; ++md) {
            if ((md == 0 && !ut) || (md == 1 && !ul) || (md == 3 && !(ut && ul))) continue;
            h264_pred(pred, 16, false, md, t, l, c, ut, ul);
            int cost = lam * (md < 2 ? 3 : 5);
            for (int b = 0; b < 16; ++b) cost += h264_satd(src + 64 * (b >> 2) + 4 * (b & 3), 16, pred + 64 * (b >> 2) + 4 * (b & 3), 16);
            if (cost < bc) { bc = cost; m.mode = (uint8_t)md; for (int k = 0; k < 256; ++k) best[k] = pred[k]; }
        }
        const int qbits = 15 + qp / 6, fq = (1 << qbits) / 3, mq = qp % 6;
        // Intra 4x4: the blocks in decoding order, each predicted from the reconstruction of the ones before it.  Top-right
        // samples exist above the macroblock (in the top-right macroblock for the last column: the x + 2 y wavefront has
        // finished it) and inside it when that block comes earlier in decoding order.
        uint8_t r4[256], tc4[16];
        int16_t l4[256];
        int c4 = lam;
        for (int b = 0; b < 16; ++b) {
            const int r = h264_blk(b), bx = r & 3, by = r >> 2, x0 = 4 * bx, y0 = 4 * by;
            auto px = [&](int xx, int yy) -> int { return xx >= 0 && yy >= 0 && xx < 16 ? r4[16 * yy + xx] : Y[(int64_t)yy * PW + xx]; };
            const bool bt = by > 0 || ut, bl = bx > 0 || ul;
            const bool btr = by == 0 ? (bx < 3 ? ut : ut && mx + 1 < a.MX) : bx < 3 && h264_blkidx(r - 3) < b;
            int e[13];
            for (int k = 0; k < 4; ++k) { e[3 - k] = bl ? px(x0 - 1, y0 + k) : 0; e[5 + k] = bt ? px(x0 + k, y0 - 1) : 0; }
            for (int k = 4; k < 8; ++k) e[5 + k] = btr ? px(x0 + k, y0 - 1) : e[8];
            e[4] = bt && bl ? px(x0 - 1, y0 - 1) : 0;
            const int pm = h264_mpm(m, ml, mt, r);
            int bcost = 0x7fffffff, bm = 2;
            uint8_t p4[16], bp[16];
            for (int md = 0; md < 9; ++md) {
                const bool need_t = md == 0 || md == 3 || md == 7 || md >= 4 && md <= 6, need_l = md == 1 || md >= 4;
                if ((need_t && !bt) || (need_l && !bl)) continue;
                h264_pred4(p4, md, e, bt, bl);
                const int cost = h264_satd(src + 16 * y0 + x0, 16, p4, 4) + lam * (md == pm ? 1 : 4);
                if (cost < bcost) { bcost = cost; bm = md; for (int k = 0; k < 16; ++k) bp[k] = p4[k]; }
            }
            m.m4[r] = (uint8_t)bm;
            c4 += bcost;
            int d[16];
            for (int j = 0; j < 4; ++j)
                for (int i = 0; i < 4; ++i) d[4 * j + i] = (int)src[16 * (y0 + j) + x0 + i] - (int)bp[4 * j + i];
            h264_fdct(d);
            int n = 0;
            for (int i = 0; i < 16; ++i) { d[i] = h264_quant(d[i], h264_mf(mq, h264_cls(i)), fq, qbits); n += d[i] != 0; }
            for (int k = 0; k < 16; ++k) l4[16 * b + k] = (int16_t)d[h264_zz(k)];
            tc4[r] = (uint8_t)n;
            for (int i = 0; i < 16; ++i) d[i] = (d[i] * h264_ls(mq, h264_cls(i))) << (qp / 6);
            h264_idct(d);
            for (int j = 0; j < 4; ++j)
                for (int i = 0; i < 4; ++i) r4[16 * (y0 + j) + x0 + i] = (uint8_t)h264_clip(bp[4 * j + i] + d[4 * j + i]);
        }
        if (c4 < bc) {
            m.mode = 5;
            m.cbp_l = 0;
            for (int r = 0; r < 16; ++r) { m.tc[r] = tc4[r]; if (tc4[r]) m.cbp_l |= (uint8_t)(1 << (h264_blkidx(r) >> 2)); }
            for (int k = 0; k < 256; ++k) { rec[k] = r4[k]; lev[k] = l4[k]; }
        } else {
        for (int k = 0; k < 16; ++k) m.m4[k] = 2;
        int dc[16], blk[16][16];
        bool any_ac = false;
        for (int r = 0; r < 16; ++r) {
            int* d = blk[r];
            for (int j = 0; j < 4; ++j)
                for (int i = 0; i < 4; ++i) {
                    const int o = 16 * (4 * (r >> 2) + j) + 4 * (r & 3) + i;
                    d[4 * j + i] = (int)src[o] - (int)best[o];
                }
            h264_fdct(d);
            dc[r] = d[0];
            for (int i = 1; i < 16; ++i) { d[i] = h264_quant(d[i], h264_mf(mq, h264_cls(i)), fq, qbits); any_ac |= d[i] != 0; }
        }
        h264_hadamard(dc);
        for (int i = 0; i < 16; ++i) dc[i] = h264_quant(dc[i] >> 1, h264_mf(mq, 0), 2 * fq, qbits + 1);
        for (int k = 0; k < 16; ++k) lev[k] = (int16_t)dc[h264_zz(k)];
        m.cbp_l = any_ac ? 15 : 0;
        for (int b = 0; b < 16; ++b) {
            const int r = h264_blk(b);
            int n = 0;
            for (int k = 1; k < 16; ++k) { lev[16 + 15 * b + k - 1] = any_ac ? (int16_t)blk[r][h264_zz(k)] : 0; n += any_ac && blk[r][h264_zz(k)] != 0; }
            m.tc[r] = (uint8_t)n;
        }
        // reconstruction: the decoder's DC inverse (8.5.10) and residual inverse (8.5.12)
        h264_hadamard(dc);
        const int ls0 = h264_ls(mq, 0);
        for (int r = 0; r < 16; ++r) {
            int* d = blk[r];
            d[0] = qp >= 12 ? (dc[r] * ls0) << (qp / 6 - 2) : (dc[r] * ls0 + (1 << (1 - qp / 6))) >> (2 - qp / 6);
            for (int i = 1; i < 16; ++i) d[i] = any_ac ? (d[i] * h264_ls(mq, h264_cls(i))) << (qp / 6) : 0;
            h264_idct(d);
            for (int j = 0; j < 4; ++j)
                for (int i = 0; i < 4; ++i) {
                    const int o = 16 * (4 * (r >> 2) + j) + 4 * (r & 3) + i;
                    rec[o] = (uint8_t)h264_clip(best[o] + d[4 * j + i]);
                }
        }
        }
    }
    // ---- chroma: one mode for Cb and Cr, least SATD + lambda bits(intra_chroma_pred_mode)
    {
        uint8_t t[2][8], l[2][8];
        int c[2];
        for (int p = 0; p < 2; ++p) {
            const uint8_t* C = h264_plane(a, f, 1 + p) + (int64_t)8 * my * (PW / 2) + 8 * mx;
            for (int k = 0; k < 8; ++k) { t[p][k] = ut ? C[k - PW / 2] : 0; l[p][k] = ul ? C[(int64_t)k * (PW / 2) - 1] : 0; }
            c[p] = ut && ul ? C[-PW / 2 - 1] : 0;
        }
        int bc = 0x7fffffff;
        m.cmode = 0;
        for (int md = 0; md < 4; ++md) {
            if ((md == 1 && !ul) || (md == 2 && !ut) || (md == 3 && !(ut && ul))) continue;
            int cost = lam * (md == 0 ? 1 : md < 3 ? 3 : 5);
            for (int p = 0; p < 2; ++p) {
                h264_pred(pred + 64 * p, 8, true, md, t[p], l[p], c[p], ut, ul);
                for (int b = 0; b < 4; ++b)
                    cost += h264_satd(src + 256 + 64 * p + 32 * (b >> 1) + 4 * (b & 1), 8, pred + 64 * p + 32 * (b >> 1) + 4 * (b & 1), 8);
            }
            if (cost < bc) { bc = cost; m.cmode = (uint8_t)md; for (int k = 0; k < 128; ++k) best[k] = pred[k]; }
        }
        const int qbits = 15 + qpc / 6, fq = (1 << qbits) / 3, mq = qpc % 6;
        int blk[2][4][16];
        bool any_dc = false, any_ac = false;
        for (int p = 0; p < 2; ++p) {
            int dc[4];
            for (int b = 0; b < 4; ++b) {
                int* d = blk[p][b];
                for (int j = 0; j < 4; ++j)
                    for (int i = 0; i < 4; ++i) {
                        const int o = 64 * p + 8 * (4 * (b >> 1) + j) + 4 * (b & 1) + i;
                        d[4 * j + i] = (int)src[256 + o] - (int)best[o];
                    }
                h264_fdct(d);
                dc[b] = d[0];
                for (int i = 1; i < 16; ++i) { d[i] = h264_quant(d[i], h264_mf(mq, h264_cls(i)), fq, qbits); any_ac |= d[i] != 0; }
            }
            const int f0 = dc[0] + dc[1] + dc[2] + dc[3], f1 = dc[0] - dc[1] + dc[2] - dc[3];
            const int f2 = dc[0] + dc[1] - dc[2] - dc[3], f3 = dc[0] - dc[1] - dc[2] + dc[3];
            const int fd[4] = {f0, f1, f2, f3};
            for (int b = 0; b < 4; ++b) {
                const int q = h264_quant(fd[b], h264_mf(mq, 0), 2 * fq, qbits + 1);
                lev[256 + 4 * p + b] = (int16_t)q;
                any_dc |= q != 0;
            }
        }
        m.cbp_c = any_ac ? 2 : any_dc ? 1 : 0;
        const int ls0 = h264_ls(mq, 0);
        for (int p = 0; p < 2; ++p) {
            const int16_t* q = lev + 256 + 4 * p;
            const int g[4] = {q[0] + q[1] + q[2] + q[3], q[0] - q[1] + q[2] - q[3], q[0] + q[1] - q[2] - q[3], q[0] - q[1] - q[2] + q[3]};
            for (int b = 0; b < 4; ++b) {
                int* d = blk[p][b];
                int n = 0;
                for (int k = 1; k < 16; ++k) {
                    const int v = any_ac ? d[h264_zz(k)] : 0;
                    lev[264 + 60 * p + 15 * b + k - 1] = (int16_t)v;
                    n += v != 0;
                }
                m.tc[16 + 4 * p + b] = (uint8_t)n;
                d[0] = ((g[b] * ls0) << (qpc / 6)) >> 1;
                for (int i = 1; i < 16; ++i) d[i] = any_ac ? (d[i] * h264_ls(mq, h264_cls(i))) << (qpc / 6) : 0;
                h264_idct(d);
                for (int j = 0; j < 4; ++j)
                    for (int i = 0; i < 4; ++i) {
                        const int o = 64 * p + 8 * (4 * (b >> 1) + j) + 4 * (b & 1) + i;
                        rec[256 + o] = (uint8_t)h264_clip(best[o] + d[4 * j + i]);
                    }
            }
        }
    }
    // ---- the exact bits; over the A.3.1 limit (or an uncodable level): I_PCM, reconstructed as the source
    BitCount cnt;
    const bool ok = h264_mb_syntax(cnt, tb, m, ml, mt, lev);
    if (!ok || cnt.n > (uint32_t)(PERF_H264_PCM_ABOVE_BITS)) {
        m.mode = 4; m.cmode = 0; m.cbp_l = 0; m.cbp_c = 0;
        for (int k = 0; k < 24; ++k) m.tc[k] = 16;
        for (int k = 0; k < 16; ++k) m.m4[k] = 2;
        for (int k = 0; k < 384; ++k) rec[k] = src[k];
        cnt.n = 0;
    }
    a.mb[mi] = m;
    a.mbits[mi] = cnt.n;
    uint8_t* Y = h264_plane(a, f, 0) + (int64_t)16 * my * PW + 16 * mx;
    for (int j = 0; j < 16; ++j)
        for (int i = 0; i < 16; ++i) Y[(int64_t)j * PW + i] = rec[16 * j + i];
    for (int p = 0; p < 2; ++p) {
        uint8_t* C = h264_plane(a, f, 1 + p) + (int64_t)8 * my * (PW / 2) + 8 * mx;
        for (int j = 0; j < 8; ++j)
            for (int i = 0; i < 8; ++i) C[(int64_t)j * (PW / 2) + i] = rec[256 + 64 * p + 8 * j + i];
    }
}

// The macroblocks of wavefront t = x + 2 y: rows y0 .. y0 + len - 1 (len may be 0 when the grid is one macroblock wide).  A
// macroblock needs its left (t - 1), top-right (t - 1), top (t - 2) and top-left (t - 3) neighbours.
__host__ __device__ __forceinline__ int h264_diag_y0(const H264Args& a)
{
    const int lo = a.t - (a.MX - 1);
    return lo > 0 ? (lo + 1) / 2 : 0;
}
__host__ __device__ __forceinline__ int h264_diag_len(const H264Args& a)
{
    const int y1 = a.t / 2 < a.MY - 1 ? a.t / 2 : a.MY - 1, n = y1 - h264_diag_y0(a) + 1;
    return n > 0 ? n : 0;
}
__host__ __device__ __forceinline__ void h264_diag_mb(const H264Args& a, const H264Tables& tb, int64_t g)
{
    const int len = h264_diag_len(a);
    const int64_t f = g / len;
    const int y = h264_diag_y0(a) + (int)(g % len);
    h264_mb(a, tb, f, a.t - 2 * y, y);
}

// ---------------------------------------------------------------- scan: one CTA per frame
struct H264ScanSmem { uint32_t len[H264_FRAME_THREADS][8]; uint32_t pre[H264_FRAME_THREADS]; uint32_t total; };

// The bits from position pos through macroblock m (I_PCM: ue(25), zero bits to a byte boundary, the samples)
__host__ __device__ __forceinline__ uint32_t h264_after(const H264Args& a, int64_t mi, uint32_t pos)
{
    if (a.mb[mi].mode != 4) return pos + a.mbits[mi];
    return ((pos + 9 + 7) & ~7u) + H264_PCM_BITS;
}

__host__ __device__ __forceinline__ void h264_scan_phase(const H264Args& a, H264ScanSmem& s, int64_t f, int p, int t)
{
    const auto [m0, m1] = thread_range<H264_FRAME_THREADS>(a.M, t);
    const int64_t base = f * a.M;
    if (p == 0) {
        for (uint32_t ph = 0; ph < 8; ++ph) {
            uint32_t pos = ph;
            for (int64_t m = m0; m < m1; ++m) pos = h264_after(a, base + m, pos);
            s.len[t][ph] = pos - ph;
        }
    } else if (p == 1) {
        if (t == 0) {
            BitCount hc;
            h264_slice_header(hc, (int)f, a.qp);
            uint32_t off = hc.n;
            for (int j = 0; j < H264_FRAME_THREADS; ++j) { s.pre[j] = off; off += s.len[j][off & 7]; }
            s.total = off + 1 + ((8 - ((off + 1) & 7)) & 7);    // rbsp_stop_one_bit, then zero bits to a byte
            a.fr[f].bits = s.total;
        }
    } else {
        uint32_t pos = s.pre[t];
        for (int64_t m = m0; m < m1; ++m) { a.moff[base + m] = pos; pos = h264_after(a, base + m, pos); }
        uint32_t* slot = (uint32_t*)(a.slots + f * a.slot);
        const uint32_t words = (s.total + 31) / 32;
        for (uint32_t i = t; i < words; i += H264_FRAME_THREADS) slot[i] = 0;
    }
}
constexpr int H264_SCAN_PHASES = 3;

// ---------------------------------------------------------------- emit: one thread per macroblock
__host__ __device__ __forceinline__ void h264_emit(const H264Args& a, const H264Tables& tb, int64_t g)
{
    const int64_t f = g / a.M, k = g % a.M;
    const int mx = (int)(k % a.MX), my = (int)(k / a.MX);
    uint32_t* slot = (uint32_t*)(a.slots + f * a.slot);
    if (k == 0) {
        MsbBits h(slot, 0);
        h264_slice_header(h, (int)f, a.qp);
        h.flush();
    }
    const H264Mb& m = a.mb[g];
    const uint32_t pos = a.moff[g];
    MsbBits w(slot, pos);
    if (m.mode == 4) {
        h264_ue(w, 25);
        w.put(0, (int)((8 - ((pos + 9) & 7)) & 7));
        const int PW = 16 * a.MX;
        const uint8_t* Y = h264_plane(a, f, 0) + (int64_t)16 * my * PW + 16 * mx;
        for (int j = 0; j < 16; ++j)
            for (int i = 0; i < 16; i += 4)
                w.put((uint32_t)Y[(int64_t)j * PW + i] << 24 | (uint32_t)Y[(int64_t)j * PW + i + 1] << 16 |
                      (uint32_t)Y[(int64_t)j * PW + i + 2] << 8 | Y[(int64_t)j * PW + i + 3], 32);
        for (int p = 0; p < 2; ++p) {
            const uint8_t* C = h264_plane(a, f, 1 + p) + (int64_t)8 * my * (PW / 2) + 8 * mx;
            for (int j = 0; j < 8; ++j)
                for (int i = 0; i < 8; i += 4)
                    w.put((uint32_t)C[(int64_t)j * (PW / 2) + i] << 24 | (uint32_t)C[(int64_t)j * (PW / 2) + i + 1] << 16 |
                          (uint32_t)C[(int64_t)j * (PW / 2) + i + 2] << 8 | C[(int64_t)j * (PW / 2) + i + 3], 32);
        }
    } else {
        h264_mb_syntax(w, tb, m, mx ? &m - 1 : nullptr, my ? &m - a.MX : nullptr, a.lev + g * H264_LEVELS);
    }
    if (k == a.M - 1) {                         // rbsp_slice_trailing_bits
        const uint32_t end = m.mode == 4 ? h264_after(a, g, pos) : pos + a.mbits[g];
        w.put(1, 1);
        w.put(0, (int)((8 - ((end + 1) & 7)) & 7));
    }
    w.flush();
}

// ---------------------------------------------------------------- nal: one CTA per frame
// Emulation prevention (7.4.1): after two zero bytes, a byte <= 3 is preceded by 0x03.  State z: the zero bytes just written
// (0, 1, 2); every thread runs its bytes from each of the three states, thread 0 chains them.
struct H264NalSmem { uint32_t ins[H264_FRAME_THREADS][3]; uint8_t st[H264_FRAME_THREADS][3]; uint32_t pre[H264_FRAME_THREADS]; uint8_t z0[H264_FRAME_THREADS]; };

__host__ __device__ __forceinline__ void h264_nal_phase(const H264Args& a, H264NalSmem& s, int64_t f, int p, int t)
{
    const uint8_t* src = a.slots + f * a.slot;
    const int64_t n = a.fr[f].bits / 8;
    const auto [i0, i1] = thread_range<H264_FRAME_THREADS>(n, t);
    if (p == 0) {
        for (int z0 = 0; z0 < 3; ++z0) {
            int z = z0;
            uint32_t k = 0;
            for (int64_t i = i0; i < i1; ++i) {
                const uint8_t b = src[i];
                if (z == 2 && b <= 3) { ++k; z = 0; }
                z = b == 0 ? (z < 2 ? z + 1 : 2) : 0;
            }
            s.ins[t][z0] = k; s.st[t][z0] = (uint8_t)z;
        }
    } else if (p == 1) {
        if (t == 0) {
            int z = 0;
            uint32_t k = 0;
            for (int j = 0; j < H264_FRAME_THREADS; ++j) { s.pre[j] = k; s.z0[j] = (uint8_t)z; k += s.ins[j][z]; z = s.st[j][z]; }
            const uint64_t nal = 1 + (uint64_t)n + k;
            a.fr[f].au = 4 + nal;
            uint8_t* o = a.nals + f * a.nal;
            o[0] = (uint8_t)(nal >> 24); o[1] = (uint8_t)(nal >> 16); o[2] = (uint8_t)(nal >> 8); o[3] = (uint8_t)nal;
            o[4] = 0x65;                        // nal_ref_idc 3, nal_unit_type 5 (IDR slice)
        }
    } else {
        uint8_t* o = a.nals + f * a.nal + 5 + i0 + s.pre[t];
        int z = s.z0[t];
        for (int64_t i = i0; i < i1; ++i) {
            const uint8_t b = src[i];
            if (z == 2 && b <= 3) { *o++ = 3; z = 0; }
            *o++ = b;
            z = b == 0 ? (z < 2 ? z + 1 : 2) : 0;
        }
    }
}
constexpr int H264_NAL_PHASES = 3;

// ---------------------------------------------------------------- finish: one CTA; write: one CTA per frame
__host__ __device__ __forceinline__ void h264_finish(const H264Args& a)
{
    uint64_t off = 0;
    for (int64_t f = 0; f < a.N; ++f) { a.fr[f].off = off; off += a.fr[f].au; }
    *a.total = off;
}

__host__ __device__ __forceinline__ void h264_write(const H264Args& a, int64_t f, int t, int nt)
{
    if (*a.total > a.out_bytes) return;
    const uint8_t* src = a.nals + f * a.nal;
    uint8_t* dst = a.out + a.fr[f].off;
    const uint64_t n = a.fr[f].au;
    for (uint64_t i = t; i < n; i += nt) dst[i] = src[i];
}

// ---------------------------------------------------------------- kernels
__device__ __forceinline__ void h264_load_tables(H264Tables& tb, const H264Args& a, int nt)
{
    for (int i = threadIdx.x; i < (int)sizeof(H264Tables); i += nt) ((uint8_t*)&tb)[i] = ((const uint8_t*)&a.tab)[i];
    __syncthreads();
}

__global__ void __launch_bounds__(H264_MB_THREADS) h264_mb_kernel(const H264Args a, int64_t n)
{
    __shared__ H264Tables tb;
    h264_load_tables(tb, a, H264_MB_THREADS);
    const int64_t g = (int64_t)blockIdx.x * H264_MB_THREADS + threadIdx.x;
    if (g < n) h264_diag_mb(a, tb, g);
}

__global__ void __launch_bounds__(H264_MB_THREADS) h264_emit_kernel(const H264Args a)
{
    __shared__ H264Tables tb;
    h264_load_tables(tb, a, H264_MB_THREADS);
    const int64_t g = (int64_t)blockIdx.x * H264_MB_THREADS + threadIdx.x;
    if (g < a.N * a.M) h264_emit(a, tb, g);
}

__global__ void h264_finish_kernel(const H264Args a) { h264_finish(a); }

__global__ void __launch_bounds__(H264_FRAME_THREADS) h264_write_kernel(const H264Args a)
{
    h264_write(a, blockIdx.x, threadIdx.x, H264_FRAME_THREADS);
}

}  // namespace perf

using namespace perf;

// ---------------------------------------------------------------- host: tables, parameter sets, layout
// Rec. ITU-T H.264 Table 9-5 (coeff_token) by nC class, [TotalCoeff][TrailingOnes]; codes are the low len bits.
static const uint8_t H264_CT_LEN[4][17][4] = {
    {{1, 0, 0, 0}, {6, 2, 0, 0}, {8, 6, 3, 0}, {9, 8, 7, 5}, {10, 9, 8, 6}, {11, 10, 9, 7}, {13, 11, 10, 8}, {13, 13, 11, 9},
     {13, 13, 13, 10}, {14, 14, 13, 11}, {14, 14, 14, 13}, {15, 15, 14, 14}, {15, 15, 15, 14}, {16, 15, 15, 15}, {16, 16, 16, 15},
     {16, 16, 16, 16}, {16, 16, 16, 16}},
    {{2, 0, 0, 0}, {6, 2, 0, 0}, {6, 5, 3, 0}, {7, 6, 6, 4}, {8, 6, 6, 4}, {8, 7, 7, 5}, {9, 8, 8, 6}, {11, 9, 9, 6}, {11, 11, 11, 7},
     {12, 11, 11, 9}, {12, 12, 12, 11}, {12, 12, 12, 11}, {13, 13, 13, 12}, {13, 13, 13, 13}, {13, 14, 13, 13}, {14, 14, 14, 13},
     {14, 14, 14, 14}},
    {{4, 0, 0, 0}, {6, 4, 0, 0}, {6, 5, 4, 0}, {6, 5, 5, 4}, {7, 5, 5, 4}, {7, 5, 5, 4}, {7, 6, 6, 4}, {7, 6, 6, 4}, {8, 7, 7, 5},
     {8, 8, 7, 6}, {9, 8, 8, 7}, {9, 9, 8, 8}, {9, 9, 9, 8}, {10, 9, 9, 9}, {10, 10, 10, 10}, {10, 10, 10, 10}, {10, 10, 10, 10}},
    {{6, 0, 0, 0}, {6, 6, 0, 0}, {6, 6, 6, 0}, {6, 6, 6, 6}, {6, 6, 6, 6}, {6, 6, 6, 6}, {6, 6, 6, 6}, {6, 6, 6, 6}, {6, 6, 6, 6},
     {6, 6, 6, 6}, {6, 6, 6, 6}, {6, 6, 6, 6}, {6, 6, 6, 6}, {6, 6, 6, 6}, {6, 6, 6, 6}, {6, 6, 6, 6}, {6, 6, 6, 6}}};
static const uint8_t H264_CT_CODE[3][17][4] = {
    {{1, 0, 0, 0}, {5, 1, 0, 0}, {7, 4, 1, 0}, {7, 6, 5, 3}, {7, 6, 5, 3}, {7, 6, 5, 4}, {15, 6, 5, 4}, {11, 14, 5, 4}, {8, 10, 13, 4},
     {15, 14, 9, 4}, {11, 10, 13, 12}, {15, 14, 9, 12}, {11, 10, 13, 8}, {15, 1, 9, 12}, {11, 14, 13, 8}, {7, 10, 9, 12}, {4, 6, 5, 8}},
    {{3, 0, 0, 0}, {11, 2, 0, 0}, {7, 7, 3, 0}, {7, 10, 9, 5}, {7, 6, 5, 4}, {4, 6, 5, 6}, {7, 6, 5, 8}, {15, 6, 5, 4}, {11, 14, 13, 4},
     {15, 10, 9, 4}, {11, 14, 13, 12}, {8, 10, 9, 8}, {15, 14, 13, 12}, {11, 10, 9, 12}, {7, 11, 6, 8}, {9, 8, 10, 1}, {7, 6, 5, 4}},
    {{15, 0, 0, 0}, {15, 14, 0, 0}, {11, 15, 13, 0}, {8, 12, 14, 12}, {15, 10, 11, 11}, {11, 8, 9, 10}, {9, 14, 13, 9}, {8, 10, 9, 8},
     {15, 14, 13, 13}, {11, 14, 10, 12}, {15, 10, 13, 12}, {11, 14, 9, 12}, {8, 10, 13, 8}, {13, 7, 9, 12}, {9, 12, 11, 10}, {5, 8, 7, 6},
     {1, 4, 3, 2}}};
// nC = -1: [TotalCoeff][TrailingOnes]
static const uint8_t H264_CDC_LEN[5][4] = {{2, 0, 0, 0}, {6, 1, 0, 0}, {6, 6, 3, 0}, {6, 7, 7, 6}, {6, 8, 8, 7}};
static const uint8_t H264_CDC_CODE[5][4] = {{1, 0, 0, 0}, {7, 1, 0, 0}, {4, 6, 1, 0}, {3, 3, 2, 5}, {2, 3, 2, 0}};
// Tables 9-7 / 9-8: total_zeros for 4x4 blocks, [TotalCoeff - 1][total_zeros]
static const uint8_t H264_TZ_LEN[15][16] = {
    {1, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 9}, {3, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 6, 6, 6, 6}, {4, 3, 3, 3, 4, 4, 3, 3, 4, 5, 5, 6, 5, 6},
    {5, 3, 4, 4, 3, 3, 3, 4, 3, 4, 5, 5, 5}, {4, 4, 4, 3, 3, 3, 3, 3, 4, 5, 4, 5}, {6, 5, 3, 3, 3, 3, 3, 3, 4, 3, 6}, {6, 5, 3, 3, 3, 2, 3, 4, 3, 6},
    {6, 4, 5, 3, 2, 2, 3, 3, 6}, {6, 6, 4, 2, 2, 3, 2, 5}, {5, 5, 3, 2, 2, 2, 4}, {4, 4, 3, 3, 1, 3}, {4, 4, 2, 1, 3}, {3, 3, 1, 2}, {2, 2, 1}, {1, 1}};
static const uint8_t H264_TZ_CODE[15][16] = {
    {1, 3, 2, 3, 2, 3, 2, 3, 2, 3, 2, 3, 2, 3, 2, 1}, {7, 6, 5, 4, 3, 5, 4, 3, 2, 3, 2, 3, 2, 1, 0}, {5, 7, 6, 5, 4, 3, 4, 3, 2, 3, 2, 1, 1, 0},
    {3, 7, 5, 4, 6, 5, 4, 3, 3, 2, 2, 1, 0}, {5, 4, 3, 7, 6, 5, 4, 3, 2, 1, 1, 0}, {1, 1, 7, 6, 5, 4, 3, 2, 1, 1, 0}, {1, 1, 5, 4, 3, 3, 2, 1, 1, 0},
    {1, 1, 1, 3, 3, 2, 2, 1, 0}, {1, 0, 1, 3, 2, 1, 1, 1}, {1, 0, 1, 3, 2, 1, 1}, {0, 1, 1, 2, 1, 3}, {0, 1, 1, 1, 1}, {0, 1, 1, 1}, {0, 1, 1}, {0, 1}};
// Table 9-9a: total_zeros for chroma DC 2x2, [TotalCoeff - 1][total_zeros]
static const uint8_t H264_CTZ_LEN[3][4] = {{1, 2, 3, 3}, {1, 2, 2, 0}, {1, 1, 0, 0}};
static const uint8_t H264_CTZ_CODE[3][4] = {{1, 1, 1, 0}, {1, 1, 0, 0}, {1, 0, 0, 0}};
// Table 9-10: run_before, [min(zerosLeft, 7) - 1][run_before]
static const uint8_t H264_RB_LEN[7][15] = {{1, 1}, {1, 2, 2}, {2, 2, 2, 2}, {2, 2, 2, 3, 3}, {2, 2, 3, 3, 3, 3}, {2, 3, 3, 3, 3, 3, 3},
                                           {3, 3, 3, 3, 3, 3, 3, 4, 5, 6, 7, 8, 9, 10, 11}};
static const uint8_t H264_RB_CODE[7][15] = {{1, 0}, {1, 1, 0}, {3, 2, 1, 0}, {3, 2, 1, 1, 0}, {3, 2, 3, 2, 1, 0}, {3, 0, 1, 3, 2, 5, 4},
                                            {7, 6, 5, 4, 3, 2, 1, 1, 1, 1, 1, 1, 1, 1, 1}};

// Table 9-4 (chroma_format_idc 1), Intra_4x4 column: coded_block_pattern of codeNum 0 .. 47
static const uint8_t H264_CBP_INTRA[48] = {47, 31, 15, 0, 23, 27, 29, 30, 7, 11, 13, 14, 39, 43, 45, 46, 16, 3, 5, 10, 12, 19, 21, 26,
                                           28, 35, 37, 42, 44, 1, 2, 4, 8, 17, 18, 20, 24, 6, 9, 22, 25, 32, 33, 34, 36, 40, 38, 41};

static void h264_tables(H264Tables& t)
{
    memset(&t, 0, sizeof(t));
    memcpy(t.ct_len, H264_CT_LEN, sizeof(t.ct_len));
    memcpy(t.ct_code, H264_CT_CODE, sizeof(H264_CT_CODE));
    for (int tc = 0; tc <= 16; ++tc)                // nC >= 8: 6-bit fixed length, (TotalCoeff - 1) << 2 | TrailingOnes; 000011 for 0
        for (int t1 = 0; t1 < 4; ++t1) t.ct_code[3][tc][t1] = (uint8_t)(tc == 0 ? 3 : ((tc - 1) << 2) | t1);
    memcpy(t.cdc_len, H264_CDC_LEN, sizeof(t.cdc_len)); memcpy(t.cdc_code, H264_CDC_CODE, sizeof(t.cdc_code));
    memcpy(t.tz_len, H264_TZ_LEN, sizeof(t.tz_len)); memcpy(t.tz_code, H264_TZ_CODE, sizeof(t.tz_code));
    memcpy(t.ctz_len, H264_CTZ_LEN, sizeof(t.ctz_len)); memcpy(t.ctz_code, H264_CTZ_CODE, sizeof(t.ctz_code));
    memcpy(t.rb_len, H264_RB_LEN, sizeof(t.rb_len)); memcpy(t.rb_code, H264_RB_CODE, sizeof(t.rb_code));
    for (int k = 0; k < 48; ++k) t.cbp_code[H264_CBP_INTRA[k]] = (uint8_t)k;
}

// Table A-1: level_idc, MaxMBPS, MaxFS (level 1b omitted: 1.1 admits the same sizes)
static const struct { int idc; int64_t mbps, fs; } H264_LEVELS_A1[] = {
    {10, 1485, 99}, {11, 3000, 396}, {12, 6000, 396}, {13, 11880, 396}, {20, 11880, 396}, {21, 19800, 792}, {22, 20250, 1620},
    {30, 40500, 1620}, {31, 108000, 3600}, {32, 216000, 5120}, {40, 245760, 8192}, {41, 245760, 8192}, {42, 522240, 8704},
    {50, 589824, 22080}, {51, 983040, 36864}, {52, 2073600, 36864}, {60, 4177920, 139264}, {61, 8355840, 139264}, {62, 16711680, 139264}};

// The smallest level whose MaxFS, MaxMBPS and frame-dimension bound (sqrt(8 MaxFS) macroblocks a side) admit the frames; 0 if none
static int h264_level(int H, int W, int fps_num, int fps_den)
{
    const int64_t MX = (W + 15) / 16, MY = (H + 15) / 16, fs = MX * MY;
    for (const auto& l : H264_LEVELS_A1)
        if (fs <= l.fs && MX * MX <= 8 * l.fs && MY * MY <= 8 * l.fs && fs * fps_num <= l.mbps * fps_den) return l.idc;
    return 0;
}

static bool h264_shape_ok(int N, int H, int W)
{
    return N >= 1 && N <= 65535 && H >= 2 && W >= 2 && H % 2 == 0 && W % 2 == 0 && H <= 16 * 1024 && W <= 16 * 1024 &&
           (int64_t)((H + 15) / 16) * ((W + 15) / 16) <= H264_MAX_MBS;
}

struct H264Layout { uint64_t plane, slot, nal, rec, mb, lev, mbits, moff, fr, total, slots, nals, bytes; };

static H264Layout h264_layout(int N, int H, int W)
{
    H264Layout l;
    const uint64_t MX = (W + 15) / 16, MY = (H + 15) / 16, M = MX * MY, n = (uint64_t)N;
    auto up = [](uint64_t v) { return (v + 255) & ~(uint64_t)255; };
    l.plane = up(384 * M);
    l.slot = up((H264_SLICE_MAX_BITS + M * H264_MB_MAX_BITS + 8 + 31) / 32 * 4);
    l.nal = up(5 + (l.slot * 3 + 1) / 2);                   // at most one 0x03 per two bytes
    l.rec = 0;
    l.mb = l.rec + n * l.plane;
    l.lev = l.mb + up(n * M * sizeof(H264Mb));
    l.mbits = l.lev + up(n * M * H264_LEVELS * 2);
    l.moff = l.mbits + up(n * M * 4);
    l.fr = l.moff + up(n * M * 4);
    l.total = l.fr + up(n * sizeof(H264Frame));
    l.slots = l.total + 256;
    l.nals = l.slots + n * l.slot;
    l.bytes = l.nals + n * l.nal;
    return l;
}

static int h264_args(H264Args& a, int N, int H, int W, void* ws, uint64_t ws_bytes)
{
    PERF_CHECK_ARG(h264_shape_ok(N, H, W), "h264 frames %d x %d x %d: needs 1 <= N <= 65535, even H and W in [2, 16384] and at most "
                   "%d macroblocks a frame", N, H, W, H264_MAX_MBS);
    PERF_CHECK_ARG(ws && (uintptr_t)ws % 16 == 0, "workspace NULL or not 16-byte aligned");
    const H264Layout l = h264_layout(N, H, W);
    PERF_CHECK_ARG(ws_bytes >= l.bytes, "workspace of %llu bytes, needs %llu", (unsigned long long)ws_bytes, (unsigned long long)l.bytes);
    memset(&a, 0, sizeof(a));
    uint8_t* w = (uint8_t*)ws;
    a.rec = w + l.rec; a.mb = (H264Mb*)(w + l.mb); a.lev = (int16_t*)(w + l.lev); a.mbits = (uint32_t*)(w + l.mbits);
    a.moff = (uint32_t*)(w + l.moff); a.fr = (H264Frame*)(w + l.fr); a.total = (uint64_t*)(w + l.total); a.slots = w + l.slots;
    a.nals = w + l.nals;
    a.N = N; a.H = H; a.W = W; a.MX = (W + 15) / 16; a.MY = (H + 15) / 16; a.M = (int64_t)a.MX * a.MY;
    a.plane = l.plane; a.slot = l.slot; a.nal = l.nal;
    return PERF_OK;
}

// The NAL unit around the RBSP that r wrote from bit 0 (rbsp_trailing_bits added here, emulation prevention included)
static int h264_nal(uint8_t* out, int cap, uint8_t header, MsbBits& r)
{
    r.put(1, 1);
    r.put(0, (int)((8 - (r.pos() & 7)) & 7));
    r.flush();
    const uint8_t* b = (const uint8_t*)r.out;
    int k = 0, z = 0;
    if (k < cap) out[k] = header;
    ++k;
    for (int i = 0; i < r.pos() / 8; ++i) {
        const uint8_t v = b[i];
        if (z == 2 && v <= 3) { if (k < cap) out[k] = 3; ++k; z = 0; }
        if (k < cap) out[k] = v;
        ++k;
        z = v == 0 ? (z < 2 ? z + 1 : 2) : 0;
    }
    return k;
}

extern "C" {
#pragma GCC visibility push(default)

int perf_h264_level(int H, int W, int fps_num, int fps_den)
{
    if (H < 2 || W < 2 || H % 2 || W % 2 || fps_num < 1 || fps_den < 1) return 0;
    return h264_level(H, W, fps_num, fps_den);
}

int perf_h264_parameter_sets(int H, int W, int fps_num, int fps_den, uint8_t* out, int out_bytes, int* sps_bytes, int* pps_bytes)
{
    PERF_CHECK_ARG(h264_shape_ok(1, H, W), "h264 frame %d x %d: needs even H and W in [2, 16384] and at most %d macroblocks", H, W,
                   H264_MAX_MBS);
    PERF_CHECK_ARG(fps_num >= 1 && fps_den >= 1 && fps_num <= 1000000 && fps_den <= 1000000, "h264 frame rate %d / %d", fps_num, fps_den);
    PERF_CHECK_ARG(out && sps_bytes && pps_bytes, "NULL pointer");
    const int level = h264_level(H, W, fps_num, fps_den);
    PERF_CHECK_ARG(level > 0, "h264 %d x %d at %d / %d fps: beyond level 6.2 (Table A-1)", H, W, fps_num, fps_den);
    const int MX = (W + 15) / 16, MY = (H + 15) / 16;
    uint32_t sps[16] = {};                                            // 64 bytes: an SPS takes at most 26
    MsbBits s(sps, 0);
    s.put(66, 8); s.put(0xC0, 8); s.put((uint32_t)level, 8);          // Constrained Baseline: constraint_set0 and 1
    h264_ue(s, 0);                                                    // seq_parameter_set_id
    h264_ue(s, 0);                                                    // log2_max_frame_num_minus4
    h264_ue(s, 2);                                                    // pic_order_cnt_type
    h264_ue(s, 0);                                                    // max_num_ref_frames
    s.put(0, 1);                                                      // gaps_in_frame_num_value_allowed_flag
    h264_ue(s, MX - 1); h264_ue(s, MY - 1);
    s.put(1, 1); s.put(1, 1);                                         // frame_mbs_only_flag, direct_8x8_inference_flag
    const bool crop = 16 * MX != W || 16 * MY != H;
    s.put(crop, 1);
    if (crop) { h264_ue(s, 0); h264_ue(s, (16 * MX - W) / 2); h264_ue(s, 0); h264_ue(s, (16 * MY - H) / 2); }
    s.put(1, 1);                                                      // vui_parameters_present_flag
    s.put(0, 1); s.put(0, 1);                                         // aspect_ratio_info, overscan_info
    s.put(1, 1); s.put(5, 3); s.put(0, 1); s.put(1, 1);               // video_signal_type: format 5, limited range, colour description
    s.put(6, 8); s.put(6, 8); s.put(6, 8);                            // BT.601 (SMPTE 170M) primaries, transfer, matrix
    s.put(0, 1);                                                      // chroma_loc_info_present_flag
    s.put(1, 1); s.put((uint32_t)fps_den, 32); s.put(2u * (uint32_t)fps_num, 32); s.put(1, 1);   // timing_info, fixed frame rate
    s.put(0, 1); s.put(0, 1); s.put(0, 1); s.put(0, 1);               // nal_hrd, vcl_hrd, pic_struct, bitstream_restriction
    uint32_t pps[16] = {};
    MsbBits p(pps, 0);
    h264_ue(p, 0); h264_ue(p, 0);                                     // pic_parameter_set_id, seq_parameter_set_id
    p.put(0, 1); p.put(0, 1);                                         // CAVLC, bottom_field_pic_order_in_frame_present_flag
    h264_ue(p, 0); h264_ue(p, 0); h264_ue(p, 0);                      // num_slice_groups_minus1, num_ref_idx_l0 / l1 minus1
    p.put(0, 1); p.put(0, 2);                                         // weighted_pred_flag, weighted_bipred_idc
    h264_se(p, 0); h264_se(p, 0); h264_se(p, 0);                      // pic_init_qp_minus26, pic_init_qs_minus26, chroma_qp_index_offset
    p.put(1, 1); p.put(0, 1); p.put(0, 1);                            // deblocking_filter_control_present, constrained_intra_pred, redundant_pic_cnt
    const int ns = h264_nal(out, out_bytes, 0x67, s);
    const int np = h264_nal(out + (ns < out_bytes ? ns : out_bytes), out_bytes - (ns < out_bytes ? ns : out_bytes), 0x68, p);
    *sps_bytes = ns; *pps_bytes = np;
    PERF_CHECK_ARG(ns + np <= out_bytes, "parameter sets of %d bytes, output of %d", ns + np, out_bytes);
    return PERF_OK;
}

uint64_t perf_h264_workspace_bytes(int N, int H, int W)
{
    return h264_shape_ok(N, H, W) ? h264_layout(N, H, W).bytes : 0;
}

int perf_h264_encode(const uint8_t* d_frames, int N, int H, int W, int qp, void* d_workspace, uint64_t workspace_bytes, void* stream)
{
    H264Args a;
    int rc = h264_args(a, N, H, W, d_workspace, workspace_bytes); if (rc) return rc;
    PERF_CHECK_ARG(d_frames, "NULL frames");
    PERF_CHECK_ARG(qp >= 0 && qp <= 51, "h264 qp %d: needs 0 <= qp <= 51", qp);
    a.rgb = d_frames; a.qp = qp;
    h264_tables(a.tab);
    const int T = a.MX + 2 * a.MY - 2;
    const cudaStream_t st = (cudaStream_t)stream;
    for (a.t = 0; a.t < T; ++a.t) {
        const int64_t n = (int64_t)N * h264_diag_len(a);
#ifdef PERF_HOST_HARNESS
        for (int64_t g = 0; g < n; ++g) h264_diag_mb(a, a.tab, g);
#else
        if (n == 0) continue;
        h264_mb_kernel<<<(unsigned)((n + H264_MB_THREADS - 1) / H264_MB_THREADS), H264_MB_THREADS, 0, st>>>(a, n);
        PERF_LAUNCH_CHECK();
#endif
    }
    rc = run_cta_phases<H264Args, H264ScanSmem, H264_FRAME_THREADS, H264_SCAN_PHASES, h264_scan_phase>(a, N, st); if (rc) return rc;
#ifdef PERF_HOST_HARNESS
    for (int64_t g = 0; g < (int64_t)N * a.M; ++g) h264_emit(a, a.tab, g);
#else
    h264_emit_kernel<<<(unsigned)(((int64_t)N * a.M + H264_MB_THREADS - 1) / H264_MB_THREADS), H264_MB_THREADS, 0, st>>>(a);
    PERF_LAUNCH_CHECK();
#endif
    rc = run_cta_phases<H264Args, H264NalSmem, H264_FRAME_THREADS, H264_NAL_PHASES, h264_nal_phase>(a, N, st); if (rc) return rc;
#ifdef PERF_HOST_HARNESS
    h264_finish(a);
#else
    h264_finish_kernel<<<1, 1, 0, st>>>(a);
    PERF_LAUNCH_CHECK();
#endif
    return PERF_OK;
}

int perf_h264_au_bytes(const void* d_workspace, uint64_t workspace_bytes, int N, int H, int W, uint64_t* d_au_bytes, void* stream)
{
    H264Args a;
    int rc = h264_args(a, N, H, W, (void*)d_workspace, workspace_bytes); if (rc) return rc;
    PERF_CHECK_ARG(d_au_bytes, "NULL pointer");
#ifdef PERF_HOST_HARNESS
    (void)stream;
    for (int f = 0; f < N; ++f) d_au_bytes[f] = a.fr[f].au;
#else
    PERF_CUDA(cudaMemcpy2DAsync(d_au_bytes, sizeof(uint64_t), &a.fr[0].au, sizeof(H264Frame), sizeof(uint64_t), N,
                                cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
#endif
    return PERF_OK;
}

int perf_h264_write(const void* d_workspace, uint64_t workspace_bytes, int N, int H, int W, uint8_t* d_out, uint64_t out_bytes,
                    uint64_t* d_total_bytes, void* stream)
{
    H264Args a;
    int rc = h264_args(a, N, H, W, (void*)d_workspace, workspace_bytes); if (rc) return rc;
    PERF_CHECK_ARG(d_out && d_total_bytes, "NULL pointer");
    a.out = d_out; a.out_bytes = out_bytes;
#ifdef PERF_HOST_HARNESS
    (void)stream;
    for (int f = 0; f < N; ++f) h264_write(a, f, 0, 1);
    *d_total_bytes = *a.total;
#else
    cudaStream_t st = (cudaStream_t)stream;
    h264_write_kernel<<<(unsigned)N, H264_FRAME_THREADS, 0, st>>>(a);
    PERF_LAUNCH_CHECK();
    PERF_CUDA(cudaMemcpyAsync(d_total_bytes, a.total, sizeof(uint64_t), cudaMemcpyDeviceToDevice, st));
#endif
    return PERF_OK;
}

int perf_h264_reconstruction(const void* d_workspace, uint64_t workspace_bytes, int N, int H, int W, uint8_t* d_yuv, void* stream)
{
    H264Args a;
    int rc = h264_args(a, N, H, W, (void*)d_workspace, workspace_bytes); if (rc) return rc;
    PERF_CHECK_ARG(d_yuv, "NULL pointer");
    const int64_t PW = 16 * (int64_t)a.MX, frame = (int64_t)H * W * 3 / 2;
    for (int64_t f = 0; f < N; ++f)
        for (int c = 0; c < 3; ++c) {
            const int64_t w = c ? W / 2 : W, h = c ? H / 2 : H, pitch = c ? PW / 2 : PW;
            uint8_t* dst = d_yuv + f * frame + (c == 0 ? 0 : (int64_t)H * W + (c - 1) * (H / 2) * (W / 2));
            const uint8_t* src = h264_plane(a, f, c);
#ifdef PERF_HOST_HARNESS
            (void)stream;
            for (int64_t y = 0; y < h; ++y) memcpy(dst + y * w, src + y * pitch, w);
#else
            PERF_CUDA(cudaMemcpy2DAsync(dst, w, src, pitch, w, h, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
#endif
        }
    return PERF_OK;
}

int perf_h264_mb_modes(const void* d_workspace, uint64_t workspace_bytes, int N, int H, int W, uint8_t* d_modes, void* stream)
{
    H264Args a;
    int rc = h264_args(a, N, H, W, (void*)d_workspace, workspace_bytes); if (rc) return rc;
    PERF_CHECK_ARG(d_modes, "NULL pointer");
    const int64_t n = (int64_t)N * a.M;
#ifdef PERF_HOST_HARNESS
    (void)stream;
    for (int64_t i = 0; i < n; ++i) memcpy(d_modes + 20 * i, &a.mb[i], 20);
#else
    PERF_CUDA(cudaMemcpy2DAsync(d_modes, 20, a.mb, sizeof(H264Mb), 20, n, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
#endif
    return PERF_OK;
}

#pragma GCC visibility pop
}
