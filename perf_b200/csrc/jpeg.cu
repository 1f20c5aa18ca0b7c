// jpeg.cu -- baseline JPEG encoder (8-bit RGB in, JFIF 4:4:4 with the Annex K Huffman tables out) with all of the coding on
// the GPU.  The restart interval is one MCU row, so every row of 8 x 8 blocks is an independent entropy-coded segment.  Five
// launches in perf_jpeg_compress and one in perf_jpeg_write:
//   bits     (one thread per MCU): colour conversion, ISLOW DCT and quantisation of the MCU's three blocks, their quantised DCs
//            and the bits of their AC codes;
//   interval (one CTA per MCU row): the DC codes' bits, the MCUs' bit offsets in the row, the row's slot zeroed;
//   emit     (one thread per MCU): the coefficients again, their Huffman codes ORed into the row's slot, word by word;
//   count    (one CTA per row): the 0xFF bytes of the row's data;
//   finish   (one CTA): the file offset of every row, the file size, the header bytes into the workspace;
//   write    (one CTA per row, one more for the header and EOI): the rows byte-stuffed into the file with their RST markers.
// perf_jpeg_file_bytes copies the file size finish computed, so a caller can size the output buffer exactly.
// Integer arithmetic only, libjpeg's default (ISLOW) path at every stage; the only atomics are integer ORs, so the bytes do not
// depend on execution order, and the host build of tests/jpeg_harness.py (-DPERF_HOST_HARNESS: each CTA's phases run over host
// arrays in a serial loop) agrees bit for bit.  Rule: perfb200.h (perf_jpeg_*).
#include "common.cuh"

namespace perf {

constexpr int JPEG_MAX_DIM = 65535;
constexpr int JPEG_MCU_MAX_BITS = 4978;         // 9 + 11 (luma DC) + 2 (11 + 11) (chroma DC) + 3 * 63 * (16 + 10) (AC)
constexpr int JPEG_HEAD_BYTES = 629;            // SOI .. SOS: 2 + 18 + 2 * 69 + 19 + 2 * (33 + 183) + 6 + 14
constexpr int JPEG_MCU_THREADS = 128;
constexpr int JPEG_ROW_THREADS = 256;
constexpr int JPEG_THREADS = 1024;

struct JpegTables {
    uint16_t qdiv[2][64];                       // 8 x the quantiser, zigzag order (luma, chroma)
    uint16_t dc_code[2][12]; uint8_t dc_len[2][12];
    uint16_t ac_code[2][256]; uint8_t ac_len[2][256];
};

struct JpegRow { uint32_t bits, nff; uint64_t off; };

struct JpegArgs {
    const uint8_t* image; uint32_t* mbits; uint32_t* moff; int16_t* mdc; JpegRow* rows; uint64_t* file_bytes; uint8_t* head;
    uint8_t* slots; uint8_t* out; uint64_t* size;
    uint64_t out_bytes;                         // perf_jpeg_write's output buffer: the file is written only if it fits
    int32_t H, W, MX, MY;                       // MCU columns (the restart interval) and rows
    int64_t M;                                  // MCUs
    uint64_t slot;                              // workspace bytes per row's unstuffed data
    JpegTables tab;
    uint8_t hdr[JPEG_HEAD_BYTES];
};

// Natural (row-major) index of zigzag position k
__host__ __device__ __forceinline__ int jpeg_zz(int k)
{
    return (uint8_t)"\x00\x01\x08\x10\x09\x02\x03\x0a\x11\x18\x20\x19\x12\x0b\x04\x05\x0c\x13\x1a\x21\x28\x30\x29\x22\x1b\x14"
                    "\x0d\x06\x07\x0e\x15\x1c\x23\x2a\x31\x38\x39\x32\x2b\x24\x1d\x16\x0f\x17\x1e\x25\x2c\x33\x3a\x3b\x34\x2d"
                    "\x26\x1f\x27\x2e\x35\x3c\x3d\x36\x2f\x37\x3e\x3f"[k];
}

// ---------------------------------------------------------------- one block: colour, DCT, quantisation
// libjpeg's jfdctint.c (LL&M, CONST_BITS 13, PASS1_BITS 2): the outputs are 8 x the orthonormal DCT.
#define JPEG_DESCALE(x, n) (((x) + (1 << ((n) - 1))) >> (n))
__host__ __device__ __forceinline__ void jpeg_fdct_1d(int32_t* d, int s, int pass)
{
    const int32_t tmp0 = d[0] + d[7 * s], tmp7 = d[0] - d[7 * s], tmp1 = d[s] + d[6 * s], tmp6 = d[s] - d[6 * s];
    const int32_t tmp2 = d[2 * s] + d[5 * s], tmp5 = d[2 * s] - d[5 * s], tmp3 = d[3 * s] + d[4 * s], tmp4 = d[3 * s] - d[4 * s];
    const int32_t tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
    const int sh = pass == 0 ? 13 - 2 : 13 + 2;
    if (pass == 0) { d[0] = (tmp10 + tmp11) * 4; d[4 * s] = (tmp10 - tmp11) * 4; }
    else { d[0] = JPEG_DESCALE(tmp10 + tmp11, 2); d[4 * s] = JPEG_DESCALE(tmp10 - tmp11, 2); }
    int32_t z1 = (tmp12 + tmp13) * 4433;
    d[2 * s] = JPEG_DESCALE(z1 + tmp13 * 6270, sh);
    d[6 * s] = JPEG_DESCALE(z1 - tmp12 * 15137, sh);
    z1 = tmp4 + tmp7;
    int32_t z2 = tmp5 + tmp6, z3 = tmp4 + tmp6, z4 = tmp5 + tmp7;
    const int32_t z5 = (z3 + z4) * 9633;
    const int32_t t4 = tmp4 * 2446, t5 = tmp5 * 16819, t6 = tmp6 * 25172, t7 = tmp7 * 12299;
    z1 *= -7373; z2 *= -20995; z3 *= -16069; z4 *= -3196;
    z3 += z5; z4 += z5;
    d[7 * s] = JPEG_DESCALE(t4 + z1 + z3, sh);
    d[5 * s] = JPEG_DESCALE(t5 + z2 + z4, sh);
    d[3 * s] = JPEG_DESCALE(t6 + z2 + z3, sh);
    d[s] = JPEG_DESCALE(t7 + z1 + z4, sh);
}

// Component c (0 Y, 1 Cb, 2 Cr) of MCU m: the quantised coefficients in zigzag order.  Samples past the right or bottom edge
// repeat the last column or row.  RGB -> YCbCr with jccolor.c's 16-bit constants (FIX(x) = round(x 2^16)); Cb and Cr round
// with 1/2 - 2^-16 so that 255 stays 255.
__host__ __device__ __forceinline__ void jpeg_block(const JpegArgs& a, const JpegTables& tb, int64_t m, int c, int32_t q[64])
{
    const int bx = (int)(m % a.MX), by = (int)(m / a.MX);
    int32_t d[64];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const int y = 8 * by + j < a.H ? 8 * by + j : a.H - 1;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const int x = 8 * bx + i < a.W ? 8 * bx + i : a.W - 1;
            const uint8_t* p = a.image + ((int64_t)y * a.W + x) * 3;
            const int32_t r = p[0], g = p[1], b = p[2];
            int32_t v;
            if (c == 0) v = (19595 * r + 38470 * g + 7471 * b + 32768) >> 16;
            else if (c == 1) v = (-11059 * r - 21709 * g + 32768 * b + (128 << 16) + 32767) >> 16;
            else v = (32768 * r - 27439 * g - 5329 * b + (128 << 16) + 32767) >> 16;
            d[8 * j + i] = v - 128;
        }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) jpeg_fdct_1d(d + 8 * j, 1, 0);
#pragma unroll
    for (int i = 0; i < 8; ++i) jpeg_fdct_1d(d + i, 8, 1);
    const uint16_t* qd = tb.qdiv[c > 0];
#pragma unroll
    for (int k = 0; k < 64; ++k) {
        const int32_t v = d[jpeg_zz(k)], dv = qd[k];
        q[k] = v < 0 ? -((-v + (dv >> 1)) / dv) : (v + (dv >> 1)) / dv;
    }
}

// The AC codes of one block (zigzag coefficients q) into the bit sink s.  libjpeg's encode_one_block: per nonzero
// coefficient, ZRL (0xF0) per 16 zeros before it, then (run, size) and the size low bits of v (v - 1 when negative); EOB
// (0x00) when the block ends in zeros.
template <class S>
__host__ __device__ __forceinline__ void jpeg_ac(const JpegTables& tb, int t, const int32_t q[64], S& s)
{
    int r = 0;
#pragma unroll
    for (int k = 1; k < 64; ++k) {
        const int32_t v = q[k];
        if (v == 0) { ++r; continue; }
        for (; r > 15; r -= 16) s.put(tb.ac_code[t][0xF0], tb.ac_len[t][0xF0]);
        const int nb = bit_width((uint32_t)(v < 0 ? -v : v)), sym = (r << 4) + nb;
        s.put(tb.ac_code[t][sym], tb.ac_len[t][sym]);
        s.put((uint32_t)(v < 0 ? v - 1 : v), nb);
        r = 0;
    }
    if (r > 0) s.put(tb.ac_code[t][0], tb.ac_len[t][0]);
}

__host__ __device__ __forceinline__ int jpeg_dc_bits(const JpegTables& tb, int t, int32_t diff)
{
    const int nb = bit_width((uint32_t)(diff < 0 ? -diff : diff));
    return tb.dc_len[t][nb] + nb;
}

// ---------------------------------------------------------------- bits / emit: one thread per MCU
__host__ __device__ __forceinline__ void jpeg_mcu_bits(const JpegArgs& a, const JpegTables& tb, int64_t m)
{
    int32_t q[64];
    BitCount bits;
    for (int c = 0; c < 3; ++c) {
        jpeg_block(a, tb, m, c, q);
        a.mdc[4 * m + c] = (int16_t)q[0];
        jpeg_ac(tb, c > 0, q, bits);
    }
    a.mdc[4 * m + 3] = 0;
    a.mbits[m] = bits.n;
}

__host__ __device__ __forceinline__ void jpeg_mcu_emit(const JpegArgs& a, const JpegTables& tb, int64_t m)
{
    const int bx = (int)(m % a.MX), by = (int)(m / a.MX);
    MsbBits w((uint32_t*)(a.slots + by * a.slot), a.moff[m]);
    int32_t q[64];
    for (int c = 0; c < 3; ++c) {
        jpeg_block(a, tb, m, c, q);
        const int32_t diff = q[0] - (bx > 0 ? a.mdc[4 * (m - 1) + c] : 0);
        const int nb = bit_width((uint32_t)(diff < 0 ? -diff : diff));
        w.put(tb.dc_code[c > 0][nb], tb.dc_len[c > 0][nb]);
        w.put((uint32_t)(diff < 0 ? diff - 1 : diff), nb);
        jpeg_ac(tb, c > 0, q, w);
    }
    if (bx == a.MX - 1) {                       // the row's last byte is padded with 1 bits
        const int pad = (int)((8 - (a.rows[by].bits & 7)) & 7);
        w.put((1u << pad) - 1u, pad);
    }
    w.flush();
}

// ---------------------------------------------------------------- interval: one CTA per MCU row
struct JpegRowSmem { uint32_t part[JPEG_ROW_THREADS], pre[JPEG_ROW_THREADS]; uint32_t total; };

__host__ __device__ __forceinline__ void jpeg_row_phase(const JpegArgs& a, JpegRowSmem& s, int64_t by, int p, int t)
{
    const auto [x0, x1] = thread_range<JPEG_ROW_THREADS>(a.MX, t);
    const int64_t m0 = by * a.MX;
    if (p == 0) {
        uint32_t sum = 0;
        for (int x = x0; x < x1; ++x) {
            const int64_t m = m0 + x;
            uint32_t b = a.mbits[m];
            for (int c = 0; c < 3; ++c) b += jpeg_dc_bits(a.tab, c > 0, a.mdc[4 * m + c] - (x > 0 ? a.mdc[4 * (m - 1) + c] : 0));
            a.mbits[m] = b;
            sum += b;
        }
        s.part[t] = sum;
    } else if (p == 1) {
        if (t == 0) {
            uint32_t b = 0;
            for (int j = 0; j < JPEG_ROW_THREADS; ++j) { s.pre[j] = b; b += s.part[j]; }
            s.total = b;
            a.rows[by].bits = b;
        }
    } else {
        uint32_t off = s.pre[t];
        for (int x = x0; x < x1; ++x) { a.moff[m0 + x] = off; off += a.mbits[m0 + x]; }
        uint32_t* slot = (uint32_t*)(a.slots + by * a.slot);
        const uint32_t words = (s.total + 7 + 31) / 32;
        for (uint32_t i = t; i < words; i += JPEG_ROW_THREADS) slot[i] = 0;
    }
}
constexpr int JPEG_ROW_PHASES = 3;

// ---------------------------------------------------------------- count: one CTA per row
struct JpegCountSmem { uint32_t n[JPEG_ROW_THREADS]; };

__host__ __device__ __forceinline__ void jpeg_count_phase(const JpegArgs& a, JpegCountSmem& s, int64_t by, int p, int t)
{
    const uint8_t* src = a.slots + by * a.slot;
    const int64_t n = (a.rows[by].bits + 7) / 8;
    if (p == 0) {
        uint32_t k = 0;
        for (int64_t i = t; i < n; i += JPEG_ROW_THREADS) k += src[i] == 0xFF;
        s.n[t] = k;
    } else if (t == 0) {
        uint32_t k = 0;
        for (int j = 0; j < JPEG_ROW_THREADS; ++j) k += s.n[j];
        a.rows[by].nff = k;
    }
}
constexpr int JPEG_COUNT_PHASES = 2;

// ---------------------------------------------------------------- finish: one CTA
struct JpegFinishSmem { uint64_t bytes[JPEG_THREADS]; uint64_t gbytes[32], gpre[32]; };

// A row's bytes in the file: its data, a 00 after every FF, and RST unless it is the last row
__host__ __device__ __forceinline__ uint64_t jpeg_row_bytes(const JpegArgs& a, int64_t i)
{
    return (a.rows[i].bits + 7) / 8 + a.rows[i].nff + (i < a.MY - 1 ? 2 : 0);
}

__host__ __device__ __forceinline__ void jpeg_finish_phase(const JpegArgs& a, JpegFinishSmem& s, int64_t, int p, int t)
{
    const auto [j0, j1] = thread_range<JPEG_THREADS>((int64_t)a.MY, t);
    const int g = t >> 5;
    if (p == 0) {
        uint64_t b = 0;
        for (int64_t i = j0; i < j1; ++i) b += jpeg_row_bytes(a, i);
        s.bytes[t] = b;
        for (int i = t; i < JPEG_HEAD_BYTES; i += JPEG_THREADS) a.head[i] = a.hdr[i];
    } else if (p == 1) {
        if (t < 32) {
            uint64_t b = 0;
            for (int j = 32 * t; j < 32 * t + 32; ++j) b += s.bytes[j];
            s.gbytes[t] = b;
        }
    } else if (p == 2) {
        if (t == 0) {
            uint64_t b = JPEG_HEAD_BYTES;
            for (int k = 0; k < 32; ++k) { s.gpre[k] = b; b += s.gbytes[k]; }
            *a.file_bytes = b + 2;
        }
    } else {
        uint64_t off = s.gpre[g];
        for (int j = 32 * g; j < t; ++j) off += s.bytes[j];
        for (int64_t i = j0; i < j1; ++i) { a.rows[i].off = off; off += jpeg_row_bytes(a, i); }
    }
}
constexpr int JPEG_FINISH_PHASES = 4;

// ---------------------------------------------------------------- write: one CTA per row, the last for the header and EOI
struct JpegWriteSmem { uint32_t n[JPEG_THREADS]; uint32_t gn[32], gpre[32]; };

__host__ __device__ __forceinline__ void jpeg_write_phase(const JpegArgs& a, JpegWriteSmem& s, int64_t by, int p, int t)
{
    const uint64_t file = *a.file_bytes;
    if (file > a.out_bytes) {                   // too small an output buffer: nothing written, size 0
        if (by == a.MY && p == 0 && t == 0) *a.size = 0;
        return;
    }
    if (by == a.MY) {
        if (p == 0) {
            for (int i = t; i < JPEG_HEAD_BYTES; i += JPEG_THREADS) a.out[i] = a.head[i];
            if (t == 0) { a.out[file - 2] = 0xFF; a.out[file - 1] = 0xD9; *a.size = file; }
        }
        return;
    }
    const uint8_t* src = a.slots + by * a.slot;
    const int64_t n = (a.rows[by].bits + 7) / 8;
    const auto [i0, i1] = thread_range<JPEG_THREADS>(n, t);
    const int g = t >> 5;
    if (p == 0) {
        uint32_t k = 0;
        for (int64_t i = i0; i < i1; ++i) k += src[i] == 0xFF;
        s.n[t] = k;
    } else if (p == 1) {
        if (t < 32) {
            uint32_t k = 0;
            for (int j = 32 * t; j < 32 * t + 32; ++j) k += s.n[j];
            s.gn[t] = k;
        }
    } else if (p == 2) {
        if (t == 0) {
            uint32_t k = 0;
            for (int j = 0; j < 32; ++j) { s.gpre[j] = k; k += s.gn[j]; }
        }
    } else {
        uint64_t o = a.rows[by].off + i0 + s.gpre[g];
        for (int j = 32 * g; j < t; ++j) o += s.n[j];
        for (int64_t i = i0; i < i1; ++i) {
            const uint8_t b = src[i];
            a.out[o++] = b;
            if (b == 0xFF) a.out[o++] = 0;
        }
        if (t == 0 && by < a.MY - 1) {
            uint8_t* r = a.out + a.rows[by].off + n + a.rows[by].nff;
            r[0] = 0xFF; r[1] = (uint8_t)(0xD0 + (by & 7));
        }
    }
}
constexpr int JPEG_WRITE_PHASES = 4;

// ---------------------------------------------------------------- kernels
__global__ void __launch_bounds__(JPEG_MCU_THREADS) jpeg_bits_kernel(const JpegArgs a)
{
    __shared__ JpegTables tb;
    for (int i = threadIdx.x; i < (int)(sizeof(JpegTables) / 2); i += JPEG_MCU_THREADS) ((uint16_t*)&tb)[i] = ((const uint16_t*)&a.tab)[i];
    __syncthreads();
    const int64_t m = (int64_t)blockIdx.x * JPEG_MCU_THREADS + threadIdx.x;
    if (m < a.M) jpeg_mcu_bits(a, tb, m);
}

__global__ void __launch_bounds__(JPEG_MCU_THREADS) jpeg_emit_kernel(const JpegArgs a)
{
    __shared__ JpegTables tb;
    for (int i = threadIdx.x; i < (int)(sizeof(JpegTables) / 2); i += JPEG_MCU_THREADS) ((uint16_t*)&tb)[i] = ((const uint16_t*)&a.tab)[i];
    __syncthreads();
    const int64_t m = (int64_t)blockIdx.x * JPEG_MCU_THREADS + threadIdx.x;
    if (m < a.M) jpeg_mcu_emit(a, tb, m);
}

}  // namespace perf

using namespace perf;

// ---------------------------------------------------------------- host: tables and header
// ITU-T T.81 Annex K: K.1 / K.2 quantisation tables (natural order), K.3 / K.5 Huffman tables (BITS, HUFFVAL)
static const uint8_t JPEG_Q[2][64] = {
    {16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55, 14, 13, 16, 24, 40, 57, 69, 56, 14, 17, 22, 29, 51, 87, 80, 62,
     18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92, 49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99},
    {17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99, 24, 26, 56, 99, 99, 99, 99, 99, 47, 66, 99, 99, 99, 99, 99, 99,
     99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99}};
static const uint8_t JPEG_DC_BITS[2][16] = {{0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0}, {0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0}};
static const uint8_t JPEG_AC_BITS[2][16] = {{0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7d}, {0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77}};
static const uint8_t JPEG_AC_VAL[2][162] = {
    {0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07, 0x22, 0x71, 0x14, 0x32, 0x81,
     0x91, 0xa1, 0x08, 0x23, 0x42, 0xb1, 0xc1, 0x15, 0x52, 0xd1, 0xf0, 0x24, 0x33, 0x62, 0x72, 0x82, 0x09, 0x0a, 0x16, 0x17, 0x18,
     0x19, 0x1a, 0x25, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x34, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48,
     0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75,
     0x76, 0x77, 0x78, 0x79, 0x7a, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99,
     0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3,
     0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe1, 0xe2, 0xe3, 0xe4, 0xe5,
     0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf1, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa},
    {0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61, 0x71, 0x13, 0x22, 0x32, 0x81, 0x08,
     0x14, 0x42, 0x91, 0xa1, 0xb1, 0xc1, 0x09, 0x23, 0x33, 0x52, 0xf0, 0x15, 0x62, 0x72, 0xd1, 0x0a, 0x16, 0x24, 0x34, 0xe1, 0x25,
     0xf1, 0x17, 0x18, 0x19, 0x1a, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45, 0x46, 0x47,
     0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74,
     0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x82, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97,
     0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba,
     0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe2, 0xe3, 0xe4,
     0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa}};

// Canonical codes (T.81 C.2) of BITS / HUFFVAL, by symbol
static void jpeg_codes(const uint8_t* bits, const uint8_t* val, uint16_t* code, uint8_t* len)
{
    int k = 0;
    uint32_t c = 0;
    for (int l = 1; l <= 16; ++l, c <<= 1)
        for (int i = 0; i < bits[l - 1]; ++i, ++k, ++c) { code[val[k]] = (uint16_t)c; len[val[k]] = (uint8_t)l; }
}

static void jpeg_tables(JpegArgs& a, int quality)
{
    memset(&a.tab, 0, sizeof(a.tab));
    const int scale = quality < 50 ? 5000 / quality : 200 - 2 * quality;         // jcparam.c jpeg_quality_scaling
    uint8_t qz[2][64];
    for (int t = 0; t < 2; ++t)
        for (int k = 0; k < 64; ++k) {
            int v = (JPEG_Q[t][jpeg_zz(k)] * scale + 50) / 100;
            v = v < 1 ? 1 : v > 255 ? 255 : v;
            qz[t][k] = (uint8_t)v;
            a.tab.qdiv[t][k] = (uint16_t)(8 * v);
        }
    uint8_t dc_val[12];
    for (int i = 0; i < 12; ++i) dc_val[i] = (uint8_t)i;
    for (int t = 0; t < 2; ++t) {
        jpeg_codes(JPEG_DC_BITS[t], dc_val, a.tab.dc_code[t], a.tab.dc_len[t]);
        jpeg_codes(JPEG_AC_BITS[t], JPEG_AC_VAL[t], a.tab.ac_code[t], a.tab.ac_len[t]);
    }
    uint8_t* h = a.hdr;
    auto b = [&](int v) { *h++ = (uint8_t)v; };
    auto w16 = [&](int v) { b(v >> 8); b(v & 255); };
    b(0xFF); b(0xD8);                                                           // SOI
    b(0xFF); b(0xE0); w16(16); b('J'); b('F'); b('I'); b('F'); b(0); b(1); b(1); b(0); w16(1); w16(1); b(0); b(0);  // APP0
    for (int t = 0; t < 2; ++t) {                                               // DQT
        b(0xFF); b(0xDB); w16(67); b(t);
        for (int k = 0; k < 64; ++k) b(qz[t][k]);
    }
    b(0xFF); b(0xC0); w16(17); b(8); w16(a.H); w16(a.W); b(3);                 // SOF0
    for (int c = 0; c < 3; ++c) { b(c + 1); b(0x11); b(c > 0); }
    for (int t = 0; t < 2; ++t)                                                 // DHT: DC t, AC t
        for (int ac = 0; ac < 2; ++ac) {
            const uint8_t* bits = ac ? JPEG_AC_BITS[t] : JPEG_DC_BITS[t];
            const int n = ac ? 162 : 12;
            b(0xFF); b(0xC4); w16(2 + 1 + 16 + n); b((ac << 4) | t);
            for (int l = 0; l < 16; ++l) b(bits[l]);
            for (int i = 0; i < n; ++i) b(ac ? JPEG_AC_VAL[t][i] : dc_val[i]);
        }
    b(0xFF); b(0xDD); w16(4); w16(a.MX);                                        // DRI
    b(0xFF); b(0xDA); w16(12); b(3);                                            // SOS
    for (int c = 0; c < 3; ++c) { b(c + 1); b(c > 0 ? 0x11 : 0x00); }
    b(0); b(63); b(0);
}

static bool jpeg_shape_ok(int H, int W) { return H >= 1 && W >= 1 && H <= JPEG_MAX_DIM && W <= JPEG_MAX_DIM; }

struct JpegLayout { uint64_t mbits, moff, mdc, rows, head, slots, slot, total; };

static JpegLayout jpeg_layout(int H, int W)
{
    JpegLayout l;
    const int64_t MX = (W + 7) / 8, MY = (H + 7) / 8, M = MX * MY;
    auto up = [](uint64_t v) { return (v + 255) & ~(uint64_t)255; };
    l.slot = ((uint64_t)MX * JPEG_MCU_MAX_BITS + 7 + 127) / 128 * 16;           // whole 16-byte units of the row's bits
    l.mbits = 0;
    l.moff = up(4 * (uint64_t)M);
    l.mdc = l.moff + up(4 * (uint64_t)M);
    l.rows = l.mdc + up(8 * (uint64_t)M);
    l.head = l.rows + up(sizeof(JpegRow) * (uint64_t)MY);
    l.slots = l.head + 1024;
    l.total = l.slots + l.slot * (uint64_t)MY;
    return l;
}

static int jpeg_args(JpegArgs& a, const uint8_t* image, int H, int W, void* ws, uint64_t ws_bytes)
{
    PERF_CHECK_ARG(jpeg_shape_ok(H, W), "jpeg image %d x %d: needs 1 <= H, W <= %d", H, W, JPEG_MAX_DIM);
    PERF_CHECK_ARG(ws && (uintptr_t)ws % 16 == 0, "workspace NULL or not 16-byte aligned");
    const JpegLayout l = jpeg_layout(H, W);
    PERF_CHECK_ARG(ws_bytes >= l.total, "workspace of %llu bytes, needs %llu", (unsigned long long)ws_bytes, (unsigned long long)l.total);
    memset(&a, 0, sizeof(a));
    uint8_t* w = (uint8_t*)ws;
    a.image = image; a.mbits = (uint32_t*)(w + l.mbits); a.moff = (uint32_t*)(w + l.moff); a.mdc = (int16_t*)(w + l.mdc);
    a.rows = (JpegRow*)(w + l.rows); a.file_bytes = (uint64_t*)(w + l.head); a.head = w + l.head + 8; a.slots = w + l.slots;
    a.H = H; a.W = W; a.MX = (W + 7) / 8; a.MY = (H + 7) / 8; a.M = (int64_t)a.MX * a.MY; a.slot = l.slot;
    return PERF_OK;
}

extern "C" {
#pragma GCC visibility push(default)

uint64_t perf_jpeg_workspace_bytes(int H, int W)
{
    return jpeg_shape_ok(H, W) ? jpeg_layout(H, W).total : 0;
}

uint64_t perf_jpeg_max_bytes(int H, int W)
{
    if (!jpeg_shape_ok(H, W)) return 0;
    const uint64_t MX = (W + 7) / 8, MY = (H + 7) / 8;
    return (uint64_t)JPEG_HEAD_BYTES + MY * (2 * ((MX * JPEG_MCU_MAX_BITS + 7) / 8) + 2) + 2;
}

int perf_jpeg_compress(const uint8_t* d_image, int H, int W, int quality, void* d_workspace, uint64_t workspace_bytes, void* stream)
{
    JpegArgs a;
    int rc = jpeg_args(a, d_image, H, W, d_workspace, workspace_bytes); if (rc) return rc;
    PERF_CHECK_ARG(d_image, "NULL image");
    PERF_CHECK_ARG(quality >= 1 && quality <= 100, "jpeg quality %d: needs 1 <= quality <= 100", quality);
    jpeg_tables(a, quality);
    const cudaStream_t st = (cudaStream_t)stream;
#ifdef PERF_HOST_HARNESS
    for (int64_t m = 0; m < a.M; ++m) jpeg_mcu_bits(a, a.tab, m);
#else
    const unsigned mcu_blocks = (unsigned)((a.M + JPEG_MCU_THREADS - 1) / JPEG_MCU_THREADS);
    jpeg_bits_kernel<<<mcu_blocks, JPEG_MCU_THREADS, 0, st>>>(a);
    PERF_LAUNCH_CHECK();
#endif
    rc = run_cta_phases<JpegArgs, JpegRowSmem, JPEG_ROW_THREADS, JPEG_ROW_PHASES, jpeg_row_phase>(a, a.MY, st); if (rc) return rc;
#ifdef PERF_HOST_HARNESS
    for (int64_t m = 0; m < a.M; ++m) jpeg_mcu_emit(a, a.tab, m);
#else
    jpeg_emit_kernel<<<mcu_blocks, JPEG_MCU_THREADS, 0, st>>>(a);
    PERF_LAUNCH_CHECK();
#endif
    rc = run_cta_phases<JpegArgs, JpegCountSmem, JPEG_ROW_THREADS, JPEG_COUNT_PHASES, jpeg_count_phase>(a, a.MY, st); if (rc) return rc;
    return run_cta_phases<JpegArgs, JpegFinishSmem, JPEG_THREADS, JPEG_FINISH_PHASES, jpeg_finish_phase>(a, 1, st);
}

int perf_jpeg_write(const void* d_workspace, uint64_t workspace_bytes, int H, int W, uint8_t* d_out, uint64_t out_bytes,
                    uint64_t* d_file_bytes, void* stream)
{
    JpegArgs a;
    int rc = jpeg_args(a, nullptr, H, W, (void*)d_workspace, workspace_bytes); if (rc) return rc;
    PERF_CHECK_ARG(d_out && d_file_bytes, "NULL pointer");
    PERF_CHECK_ARG(out_bytes >= (uint64_t)JPEG_HEAD_BYTES + 2, "output of %llu bytes, a JPEG takes more than %d",
                   (unsigned long long)out_bytes, JPEG_HEAD_BYTES + 2);
    a.out = d_out; a.out_bytes = out_bytes; a.size = d_file_bytes;
    return run_cta_phases<JpegArgs, JpegWriteSmem, JPEG_THREADS, JPEG_WRITE_PHASES, jpeg_write_phase>(a, a.MY + 1,
                                                                                                    (cudaStream_t)stream);
}

int perf_jpeg_file_bytes(const void* d_workspace, uint64_t workspace_bytes, int H, int W, uint64_t* d_file_bytes, void* stream)
{
    JpegArgs a;
    int rc = jpeg_args(a, nullptr, H, W, (void*)d_workspace, workspace_bytes); if (rc) return rc;
    PERF_CHECK_ARG(d_file_bytes, "NULL pointer");
#ifdef PERF_HOST_HARNESS
    (void)stream;
    *d_file_bytes = *a.file_bytes;
#else
    PERF_CUDA(cudaMemcpyAsync(d_file_bytes, a.file_bytes, sizeof(uint64_t), cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
#endif
    return PERF_OK;
}

#pragma GCC visibility pop
}
