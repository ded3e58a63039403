// Baseline JPEG decoding on the device, byte-identical to libjpeg-turbo's default decompression (what cv2.imdecode(buf,
// IMREAD_UNCHANGED) and mmcv.imread(name, 'unchanged') run): ISLOW integer IDCT with its range-limit table, h2v2 fancy
// upsampling, integer YCbCr -> BGR tables.  The CPU restatement is oracle/jpeg_decode.py.
//
// Host: the markers are parsed and every component's Huffman lookup tables and natural-order quantisation table are built
// into one descriptor per image; descriptors and entropy-coded segments go to the device in one upload from a pinned staging
// buffer, guarded by an event.  The end of the segment is the EOI marker at the end of the file, so the host never scans it.
//
// Device, all images of a call in the same three launches:
//   jpeg_entropy_kernel  one 1024-thread block per image: removes the FF00 stuffing, the RSTn markers (recording every restart
//                        interval's start) and the FF fill bytes before RSTn and EOI, cuts each interval into kSubBits-bit
//                        subsequences and decodes them with self-synchronising Huffman decoding (Weissenberger & Schmidt, ICPP
//                        2018): every subsequence decodes from a guessed start state (bit position, block of the MCU, zig-zag
//                        index) to the first codeword boundary at or past its end; then, until no start changes, each takes its
//                        predecessor's exit state as its start and decodes again.  An interval's first subsequence starts from
//                        the true state, so at convergence every start is a true codeword boundary (the worst case is serial
//                        decoding, never a wrong one).  A scan of the per-subsequence block counts places every block; the
//                        coefficients go to an int16 block array in decode order and the DC differences are summed by a
//                        segmented scan that restarts at every interval.
//   jpeg_idct_kernel     dequantisation + ISLOW IDCT (jidctint.c), 8 threads per block, into per-component sample planes.
//   jpeg_color_kernel    h2v2 fancy upsampling (4:2:0) + YCbCr -> BGR, interleaved uint8 straight into the frame buffer.
// Corrupt data (an invalid code, a run past coefficient 63, an interval that ends early or late, a marker inside the scan) never
// reads or writes out of bounds: the image's status word is set and its coefficients are zeroed.
#include <cuda_runtime.h>

#include <cstring>
#include <string>
#include <vector>

#include "../../include/occ_b200.h"
#include "common.cuh"
#include "jpeg.cuh"

namespace occ {
namespace {

constexpr int kThreads = 1024;          // jpeg_entropy_kernel block
constexpr int kSubBits = 1024;          // subsequence length of the self-synchronising decoder
constexpr int kPad = 16;                // 0xFF bytes after every unstuffed segment (the bit reader reads 8 bytes ahead)

// Huffman table of one component: a 9-bit lookup (length << 8 | symbol, 0 = longer code) and the canonical maxcode / value
// offset per length for codes of 10..16 bits (jdhuff.c's derived table)
struct HuffTable {
    uint16_t lut[512];
    int32_t maxcode[17];
    int32_t valoff[17];
    uint8_t val[256];
};

struct JpegImage {
    int h, w, sub;                      // sub 2 = 4:2:0, 1 = 4:4:4
    int mcux, mcuy, bpm;                // MCUs per row / column, blocks per MCU (6 or 3)
    int ri, n_iv;                       // MCUs per restart interval (all of them without DRI), intervals
    int seg_len, n_sub_cap;
    int64_t seg_off;                    // entropy-coded bytes in the upload, and the unstuffed bytes in `unst`
    int64_t iv_off, sub_off;            // int32 [n_iv + 1] interval starts / first subsequences; subsequence arrays
    int64_t coef_off;                   // first block (64 int16) in decode order
    int64_t plane_off[3];               // component sample planes, (mcuy * 8 * s) x (mcux * 8 * s) bytes, s = sub for Y
    int64_t out_off;                    // h x w x 3 bytes in the output
    uint16_t q[3][64];                  // natural order
    HuffTable dc[3], ac[3];
};

struct Bufs {
    const JpegImage* img;
    const uint8_t* in;
    uint8_t* unst;
    int32_t *iv, *sub_first, *sub_iv, *cnt;
    uint2 *st, *ex, *nst;               // decoder states: x = bit position, y = block << 8 | zig-zag index
    int16_t* coef;
    uint8_t* planes;
    uint8_t* out;
    int32_t* status;                    // per image, 0 = decoded
};

constexpr int kZigzag[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                             41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                             30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};
__constant__ uint8_t c_zigzag[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                                     41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                                     30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

// ---------------------------------------------------------------------------------------------------------------- host
struct Prepared {
    JpegImage im;
    const uint8_t* seg;
};

int build_huff(const uint8_t* bits, const uint8_t* vals, int nvals, bool dc, HuffTable& t)
{
    memset(&t, 0, sizeof(t));
    int code = 0, k = 0;
    for (int l = 1; l <= 16; ++l) {
        t.maxcode[l] = -1;
        // jdhuff.c's rule: the codes of length l must fit in l bits, and the all-ones code is reserved (checked before the
        // lookup is filled, so an over-subscribed table is refused without writing past it)
        OCC_CHECK(code + bits[l - 1] < (1 << l), "corrupt Huffman table (over-subscribed code lengths)");
        OCC_CHECK(k + bits[l - 1] <= nvals, "corrupt Huffman table");
        if (bits[l - 1]) {
            t.valoff[l] = k - code;
            for (int i = 0; i < bits[l - 1]; ++i, ++code, ++k) {
                if (l <= 9)
                    for (int f = 0; f < (1 << (9 - l)); ++f) t.lut[(code << (9 - l)) | f] = (uint16_t)(l << 8 | vals[k]);
            }
            t.maxcode[l] = code - 1;
        }
        code <<= 1;
    }
    OCC_CHECK(k == nvals && k <= 256, "corrupt Huffman table");
    memcpy(t.val, vals, nvals);
    if (dc)
        for (int i = 0; i < nvals; ++i) OCC_CHECK(vals[i] <= 15, "corrupt DC Huffman table");
    return 0;
}

inline int be16(const uint8_t* p) { return p[0] << 8 | p[1]; }

// The header of one file -> descriptor (tables, geometry); the entropy-coded segment runs from the end of the SOS header to the
// EOI marker that ends the file.
int parse_jpeg(const uint8_t* d, int64_t n, Prepared& out)
{
    OCC_CHECK(d != nullptr && n >= 4 && d[0] == 0xFF && d[1] == 0xD8, "not a JPEG file (no SOI marker)");
    static thread_local std::vector<HuffTable> ht;
    ht.assign(8, HuffTable());
    bool have_q[4] = {}, have_h[8] = {};
    uint16_t qt[4][64];
    int restart = 0, comp_id[3] = {}, comp_q[3] = {};
    bool sof = false;
    JpegImage& im = out.im;
    memset(&im, 0, sizeof(im));
    int64_t p = 2;
    for (;;) {
        while (p + 1 < n && d[p] == 0xFF && d[p + 1] == 0xFF) ++p;            // fill bytes
        OCC_CHECK(p + 4 <= n, "truncated file (header)");
        OCC_CHECK(d[p] == 0xFF, "corrupt header (marker expected)");
        const int m = d[p + 1], len = be16(d + p + 2);
        OCC_CHECK(len >= 2 && p + 2 + len <= n, "truncated file (header)");
        const uint8_t* s = d + p + 4;
        const int sl = len - 2;
        OCC_CHECK(!(m == 0xC2 || m == 0xC6 || m == 0xCA || m == 0xCE), "progressive JPEG is not supported");
        OCC_CHECK(!(m == 0xC9 || m == 0xCB || m == 0xCC || m == 0xCD || m == 0xCF), "arithmetic coding is not supported");
        OCC_CHECK(!(m == 0xC3 || m == 0xC5 || m == 0xC7), "lossless / hierarchical JPEG is not supported");
        OCC_CHECK(!(m == 0xEE && sl >= 5 && memcmp(s, "Adobe", 5) == 0), "Adobe-transform (APP14) files are not supported");
        OCC_CHECK(m != 0xD9, "no scan in the file");
        if (m == 0xC0 || m == 0xC1) {
            OCC_CHECK(sl >= 6, "corrupt frame header");
            OCC_CHECK(s[0] == 8, std::to_string(s[0]) + "-bit samples are not supported");
            const int nc = s[5];
            OCC_CHECK(nc != 1, "grayscale JPEG is not supported");
            OCC_CHECK(nc == 3, std::to_string(nc) + "-component (CMYK) JPEG is not supported");
            OCC_CHECK(sl >= 15, "corrupt frame header");
            int hv[3][2];
            for (int c = 0; c < 3; ++c) {
                comp_id[c] = s[6 + 3 * c];
                hv[c][0] = s[7 + 3 * c] >> 4; hv[c][1] = s[7 + 3 * c] & 15;
                comp_q[c] = s[8 + 3 * c];
                OCC_CHECK(comp_q[c] < 4, "corrupt frame header");
            }
            OCC_CHECK(!(comp_id[0] == 'R' && comp_id[1] == 'G' && comp_id[2] == 'B'),
                      "RGB (untransformed) JPEG is not supported");
            bool c11 = true;
            for (int c = 1; c < 3; ++c) c11 = c11 && hv[c][0] == 1 && hv[c][1] == 1;
            if (c11 && hv[0][0] == 2 && hv[0][1] == 2) im.sub = 2;
            else if (c11 && hv[0][0] == 1 && hv[0][1] == 1) im.sub = 1;
            else OCC_CHECK(false, "chroma sampling Y " + std::to_string(hv[0][0]) + "x" + std::to_string(hv[0][1]) + ", Cb " +
                                      std::to_string(hv[1][0]) + "x" + std::to_string(hv[1][1]) + ", Cr " +
                                      std::to_string(hv[2][0]) + "x" + std::to_string(hv[2][1]) +
                                      " is not supported (only 4:2:0 and 4:4:4)");
            im.h = be16(s + 1);
            im.w = be16(s + 3);
            OCC_CHECK(im.h > 0 && im.w > 0, "empty image (or a DNL marker, which is not supported)");
            sof = true;
        } else if (m == 0xDB) {
            for (int q = 0; q < sl;) {
                OCC_CHECK((s[q] >> 4) == 0, "16-bit quantisation tables are not supported");
                const int tq = s[q] & 15;
                OCC_CHECK(tq < 4 && q + 65 <= sl, "corrupt quantisation table");
                for (int i = 0; i < 64; ++i) qt[tq][kZigzag[i]] = s[q + 1 + i];
                have_q[tq] = true;
                q += 65;
            }
        } else if (m == 0xC4) {
            for (int q = 0; q < sl;) {
                OCC_CHECK(q + 17 <= sl, "corrupt Huffman table");
                const int tc = s[q] >> 4, th = s[q] & 15;
                OCC_CHECK(tc <= 1 && th < 4, "corrupt Huffman table");
                int nv = 0;
                for (int i = 0; i < 16; ++i) nv += s[q + 1 + i];
                OCC_CHECK(q + 17 + nv <= sl, "corrupt Huffman table");
                if (build_huff(s + q + 1, s + q + 17, nv, tc == 0, ht[tc * 4 + th])) return 1;
                have_h[tc * 4 + th] = true;
                q += 17 + nv;
            }
        } else if (m == 0xDD) {
            OCC_CHECK(sl >= 2, "corrupt restart interval");
            restart = be16(s);
        } else if (m == 0xDA) {
            OCC_CHECK(sof, "scan before the frame header");
            OCC_CHECK(sl >= 1 && s[0] == 3, "several scans (non-interleaved components) are not supported");
            OCC_CHECK(sl >= 10, "corrupt scan header");
            for (int c = 0; c < 3; ++c) {
                OCC_CHECK(s[1 + 2 * c] == comp_id[c], "scan components differ from the frame components");
                const int td = s[2 + 2 * c] >> 4, ta = s[2 + 2 * c] & 15;
                OCC_CHECK(td < 4 && ta < 4 && have_h[td] && have_h[4 + ta], "scan uses an undefined Huffman table");
                OCC_CHECK(have_q[comp_q[c]], "frame uses an undefined quantisation table");
                im.dc[c] = ht[td];
                im.ac[c] = ht[4 + ta];
                memcpy(im.q[c], qt[comp_q[c]], sizeof(im.q[c]));
            }
            OCC_CHECK(s[7] == 0 && s[8] == 63 && s[9] == 0, "progressive scan parameters are not supported");
            const int64_t start = p + 2 + len;
            // the scan ends at the last EOI marker of the file: bytes after it are ignored, as libjpeg ignores them (a trailer
            // that itself holds FF D9 would put its bytes into the scan, which the device then reports as corrupt)
            int64_t eoi = n - 2;
            while (eoi >= start && !(d[eoi] == 0xFF && d[eoi + 1] == 0xD9)) --eoi;
            OCC_CHECK(eoi >= start, "truncated file (no EOI marker after the scan)");
            n = eoi + 2;
            // bit positions are 32-bit on the device
            OCC_CHECK(n - 2 - start < (int64_t)1 << 28, "scan larger than 256 MiB");
            out.seg = d + start;
            im.seg_len = (int)(n - 2 - start);
            const int ms = 8 * im.sub;
            im.mcux = (im.w + ms - 1) / ms;
            im.mcuy = (im.h + ms - 1) / ms;
            im.bpm = im.sub == 2 ? 6 : 3;
            const int mcus = im.mcux * im.mcuy;
            im.ri = restart > 0 && restart < mcus ? restart : mcus;
            im.n_iv = (mcus + im.ri - 1) / im.ri;
            im.n_sub_cap = im.n_iv + (int)(((int64_t)im.seg_len * 8 + kSubBits - 1) / kSubBits);
            return 0;
        }
        p += 2 + len;
    }
}

// ---------------------------------------------------------------------------------------------------------------- device
__device__ __forceinline__ uint32_t load_be32(const uint8_t* p)      // p 4-byte aligned
{
    return __byte_perm(*reinterpret_cast<const uint32_t*>(p), 0, 0x0123);
}

// 32 bits of the stream starting at bit `pos`
__device__ __forceinline__ uint32_t peek32(const uint8_t* s, uint32_t pos)
{
    const uint8_t* w = s + ((pos >> 5) << 2);
    return __funnelshift_l(load_be32(w + 4), load_be32(w), pos & 31);
}

__device__ __forceinline__ int extend(int v, int s) { return s && v < (1 << (s - 1)) ? v - (1 << s) + 1 : v; }

struct Layout {
    int bpm;
    __device__ int comp(int blk) const { return bpm == 6 ? (blk < 4 ? 0 : blk - 3) : blk; }
};

// One Huffman code + its extra bits from state (pos, blk, zz).  `coef` (the block being decoded, zig-zag positions mapped to
// natural order; the DC as its difference) receives the value when non-null.  Returns false on corrupt data; the state always
// advances deterministically.
__device__ __forceinline__ bool decode_symbol(const uint8_t* s, const HuffTable* dc, const HuffTable* ac, Layout L,
                                              uint32_t& pos, int& blk, int& zz, int16_t* coef)
{
    const int c = L.comp(blk);
    const HuffTable& t = zz == 0 ? dc[c] : ac[c];
    const uint32_t win = peek32(s, pos);
    const uint32_t p16 = win >> 16;
    int len = 0, sym = 0;
    const uint16_t e = t.lut[p16 >> 7];
    if (e) {
        len = e >> 8;
        sym = e & 255;
    } else {
        for (int l = 10; l <= 16; ++l) {
            const int code = (int)(p16 >> (16 - l));
            if (code <= t.maxcode[l]) { len = l; sym = t.val[code + t.valoff[l]]; break; }
        }
        if (len == 0) { pos += 1; return false; }
    }
    bool ok = true;
    if (zz == 0) {
        const int sz = sym;
        if (coef) coef[0] = (int16_t)extend(sz ? (int)((win << len) >> (32 - sz)) : 0, sz);
        pos += len + sz;
        zz = 1;
    } else {
        const int r = sym >> 4, sz = sym & 15;
        if (sz == 0) {
            zz = r == 15 ? zz + 16 : 64;
            pos += len;
        } else {
            zz += r;
            if (zz > 63) {
                ok = false;
            } else if (coef) {
                coef[c_zigzag[zz]] = (int16_t)extend((int)((win << len) >> (32 - sz)), sz);
            }
            pos += len + sz;
            zz = zz > 63 ? 64 : zz + 1;
        }
    }
    if (zz >= 64) {
        ok = ok && zz == 64;
        zz = 0;
        blk = blk + 1 == L.bpm ? 0 : blk + 1;
    }
    return ok;
}

__device__ __forceinline__ uint2 pack_state(uint32_t pos, int blk, int zz) { return make_uint2(pos, (uint32_t)(blk << 8 | zz)); }

// decode from `st` to the first codeword boundary at or past bit `end` -> exit state; blocks started on the way
__device__ uint2 run_sub(const uint8_t* s, const HuffTable* dc, const HuffTable* ac, Layout L, uint2 st, uint32_t end,
                         int& nblk)
{
    uint32_t pos = st.x;
    int blk = st.y >> 8, zz = st.y & 255, n = 0;
    while (pos < end) {
        n += zz == 0;
        decode_symbol(s, dc, ac, L, pos, blk, zz, nullptr);
    }
    nblk = n;
    return pack_state(pos, blk, zz);
}

// exclusive block-wide sum over kThreads threads; *total receives the sum
__device__ int block_scan(int v, int* sh, int* total)
{
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    int x = v;
    for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
    }
    if (lane == 31) sh[wid] = x;
    __syncthreads();
    if (wid == 0) {
        int w = sh[lane];
        for (int o = 1; o < 32; o <<= 1) {
            const int y = __shfl_up_sync(0xffffffffu, w, o);
            if (lane >= o) w += y;
        }
        sh[lane] = w;
    }
    __syncthreads();
    const int r = x - v + (wid ? sh[wid - 1] : 0);
    *total = sh[31];
    __syncthreads();
    return r;
}

// segmented exclusive-carry scan: (reset, sum) pairs, combine (a then b) = (a.f | b.f, b.f ? b.s : a.s + b.s)
__device__ int block_seg_scan(int f, int v, int* shf, int* shv, int& carry_f)
{
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    int xf = f, xv = v;
    for (int o = 1; o < 32; o <<= 1) {
        const int yf = __shfl_up_sync(0xffffffffu, xf, o), yv = __shfl_up_sync(0xffffffffu, xv, o);
        if (lane >= o) { xv = xf ? xv : xv + yv; xf |= yf; }
    }
    if (lane == 31) { shf[wid] = xf; shv[wid] = xv; }
    __syncthreads();
    if (wid == 0) {
        int wf = shf[lane], wv = shv[lane];
        for (int o = 1; o < 32; o <<= 1) {
            const int yf = __shfl_up_sync(0xffffffffu, wf, o), yv = __shfl_up_sync(0xffffffffu, wv, o);
            if (lane >= o) { wv = wf ? wv : wv + yv; wf |= yf; }
        }
        shf[lane] = wf; shv[lane] = wv;
    }
    __syncthreads();
    // exclusive prefix of this thread = inclusive prefix of the previous thread
    int pf = __shfl_up_sync(0xffffffffu, xf, 1), pv = __shfl_up_sync(0xffffffffu, xv, 1);
    if (lane == 0) { pf = 0; pv = 0; }
    if (wid > 0) {
        const int wf = shf[wid - 1], wv = shv[wid - 1];
        pv = pf ? pv : pv + wv;
        pf |= wf;
    }
    carry_f = pf;
    __syncthreads();
    return pv;
}

__device__ __forceinline__ bool is_rst(uint8_t b) { return b >= 0xD0 && b <= 0xD7; }

enum { kKeep, kRst, kDrop };

// Calls f(kind, i) for every byte i in [b0, b1) of the entropy-coded segment in[0, n): kKeep for a data byte (the FF of FF00
// included), kRst for the FF of an RSTn marker, kDrop for the 00 of FF00, an RSTn byte and a fill byte.  A marker may be
// preceded by any number of FF fill bytes (T.81 B.1.1.2): a run of FF bytes that ends in an RSTn byte, or at the end of the
// segment (the EOI marker follows), is fill plus that marker.  Any other FF not followed by 00, FF FF 00 included, sets `bad`.
// A run that crosses the chunk is classified from its own bytes, so every thread gives the bytes of its chunk the same kind.
template <class F>
__device__ __forceinline__ void for_each_byte(const uint8_t* in, int n, int b0, int b1, int& bad, F f)
{
    for (int i = b0; i < b1;) {
        if (in[i] != 0xFF) {
            f(i > 0 && in[i - 1] == 0xFF ? kDrop : kKeep, i);
            ++i;
            continue;
        }
        int k = i + 1;                                               // the run of FF bytes containing i ends at k - 1
        while (k < n && in[k] == 0xFF) ++k;
        const bool single = k - 1 == 0 || in[k - 2] != 0xFF;
        int last;                                                    // what the run's last FF is
        if (k == n) last = kDrop;
        else if (is_rst(in[k])) last = kRst;
        else if (in[k] == 0 && single) last = kKeep;
        else { bad = 1; last = kDrop; }
        for (; i < min(k, b1); ++i) f(i == k - 1 ? last : kDrop, i);
    }
}

__global__ void __launch_bounds__(kThreads, 1) jpeg_entropy_kernel(Bufs B)
{
    const JpegImage& im = B.img[blockIdx.x];
    __shared__ HuffTable s_dc[3], s_ac[3];
    __shared__ int sh[32], sh2[32];
    __shared__ int s_bad, s_changed;
    const int tid = threadIdx.x;
    for (int i = tid; i < (int)(sizeof(HuffTable) / 4); i += kThreads)
        for (int c = 0; c < 3; ++c) {
            reinterpret_cast<int*>(&s_dc[c])[i] = reinterpret_cast<const int*>(&im.dc[c])[i];
            reinterpret_cast<int*>(&s_ac[c])[i] = reinterpret_cast<const int*>(&im.ac[c])[i];
        }
    if (tid == 0) s_bad = 0;
    const Layout L{im.bpm};
    const uint8_t* in = B.in + im.seg_off;
    uint8_t* us = B.unst + im.seg_off;
    int32_t* iv = B.iv + im.iv_off;
    const int n = im.seg_len, n_iv = im.n_iv;
    const int64_t nblocks = (int64_t)im.mcux * im.mcuy * im.bpm;
    int16_t* coef = B.coef + im.coef_off * 64;
    // zero the coefficients (the decoder writes the non-zero ones only)
    for (int64_t i = tid; i < nblocks * 8; i += kThreads) reinterpret_cast<int4*>(coef)[i] = make_int4(0, 0, 0, 0);

    // ---- 1. unstuffing: each thread a contiguous chunk of bytes; byte i is kept unless it is the 00 of FF00, part of a
    // marker or a fill byte.  RSTn markers record the start of the next interval and must count 0..7 in order.
    {
        const int chunk = (n + kThreads - 1) / kThreads;
        const int b0 = min(n, tid * chunk), b1 = min(n, b0 + chunk);
        int keep = 0, rst = 0, bad = 0;
        for_each_byte(in, n, b0, b1, bad, [&](int kind, int) { keep += kind == kKeep; rst += kind == kRst; });
        int tk, tr;
        int ok = block_scan(keep, sh, &tk);
        int orr = block_scan(rst, sh, &tr);
        for_each_byte(in, n, b0, b1, bad, [&](int kind, int i) {
            if (kind == kKeep) {
                us[ok++] = in[i];
            } else if (kind == kRst) {
                if (orr + 1 < n_iv) iv[orr + 1] = ok;
                if ((in[i + 1] & 7) != (orr & 7)) bad = 1;
                ++orr;
            }
        });
        if (bad) s_bad = 1;
        if (tid < kPad) us[tk + tid] = 0xFF;
        if (tid == 0) {
            iv[0] = 0;
            iv[n_iv] = tk;
            if (tr != n_iv - 1) s_bad = 1;
        }
    }
    __syncthreads();
    if (s_bad) {
        if (tid == 0) B.status[blockIdx.x] = 1;
        return;                                                      // coefficients stay zero
    }
    // ---- 2. subsequences: interval r gets max(1, ceil(bits / kSubBits)) of them
    int32_t* sub_first = B.sub_first + im.iv_off;
    int32_t* sub_iv = B.sub_iv + im.sub_off;
    uint2* st = B.st + im.sub_off;
    uint2* ex = B.ex + im.sub_off;
    uint2* nst = B.nst + im.sub_off;
    int32_t* cnt = B.cnt + im.sub_off;
    int n_sub = 0;
    {
        const int chunk = (n_iv + kThreads - 1) / kThreads;
        const int r0 = min(n_iv, tid * chunk), r1 = min(n_iv, r0 + chunk);
        int k = 0;
        for (int r = r0; r < r1; ++r) k += max(1, (8 * (iv[r + 1] - iv[r]) + kSubBits - 1) / kSubBits);
        int o = block_scan(k, sh, &n_sub);
        for (int r = r0; r < r1; ++r) {
            sub_first[r] = o;
            const int kr = max(1, (8 * (iv[r + 1] - iv[r]) + kSubBits - 1) / kSubBits);
            for (int j = 0; j < kr; ++j) sub_iv[o + j] = r;
            o += kr;
        }
        if (tid == 0) sub_first[n_iv] = n_sub;
    }
    __syncthreads();
    // ---- 3. first decode of every subsequence from its guessed start
    auto bounds = [&](int j, uint32_t& s0, uint32_t& e0) {
        const int r = sub_iv[j];
        s0 = 8u * iv[r] + (uint32_t)(j - sub_first[r]) * kSubBits;
        e0 = min(s0 + kSubBits, 8u * iv[r + 1]);
    };
    for (int j = tid; j < n_sub; j += kThreads) {
        uint32_t s0, e0;
        bounds(j, s0, e0);
        const uint2 g = pack_state(s0, 0, 0);
        int k;
        st[j] = g;
        ex[j] = run_sub(us, s_dc, s_ac, L, g, e0, k);
        cnt[j] = k;
    }
    // ---- 4. synchronise: take the predecessor's exit state until no start changes
    for (;;) {
        __syncthreads();
        if (tid == 0) s_changed = 0;
        for (int j = tid; j < n_sub; j += kThreads) {
            uint2 ns = make_uint2(0xffffffffu, 0);
            if (j != sub_first[sub_iv[j]]) {
                const uint2 x = ex[j - 1], s = st[j];
                if (x.x != s.x || x.y != s.y) ns = x;
            }
            nst[j] = ns;
        }
        __syncthreads();
        for (int j = tid; j < n_sub; j += kThreads) {
            const uint2 ns = nst[j];
            if (ns.x == 0xffffffffu) continue;
            uint32_t s0, e0;
            bounds(j, s0, e0);
            int k;
            st[j] = ns;
            ex[j] = run_sub(us, s_dc, s_ac, L, ns, e0, k);
            cnt[j] = k;
            s_changed = 1;
        }
        __syncthreads();
        if (!s_changed) break;
    }
    // ---- 5. block base of every subsequence: exclusive scan of the counts within its interval (the last subsequence of an
    // interval is counted as 0: it may decode the padding bits into blocks that do not exist)
    int32_t* base = reinterpret_cast<int32_t*>(nst);                  // nst is free now
    {
        const int chunk = (n_sub + kThreads - 1) / kThreads;
        const int j0 = min(n_sub, tid * chunk), j1 = min(n_sub, j0 + chunk);
        auto is_last = [&](int j) { return j + 1 == n_sub || sub_iv[j + 1] != sub_iv[j]; };
        int k = 0;
        for (int j = j0; j < j1; ++j) k += is_last(j) ? 0 : cnt[j];
        int tot;
        int o = block_scan(k, sh, &tot);
        for (int j = j0; j < j1; ++j) { base[j] = o; o += is_last(j) ? 0 : cnt[j]; }
    }
    __syncthreads();
    // ---- 6. final decode: every subsequence writes the coefficients of the blocks it decodes; the last one of an interval
    // stops after the interval's last block and must end in the interval's padding bits
    const int mcus = im.mcux * im.mcuy;
    for (int j = tid; j < n_sub; j += kThreads) {
        const int r = sub_iv[j];
        const int64_t iv_blk0 = (int64_t)r * im.ri * im.bpm;
        const int need = min(im.ri, mcus - r * im.ri) * im.bpm;
        const bool last = j + 1 == n_sub || sub_iv[j + 1] != r;
        uint32_t s0, e0;
        bounds(j, s0, e0);
        uint32_t pos = st[j].x;
        int blk = st[j].y >> 8, zz = st[j].y & 255;
        int b = base[j] - base[sub_first[r]];                           // blocks of the interval started before (a started
                                                                        // block, zz != 0, is block b - 1 and continues here)
        bool bad = false;
        for (;;) {
            if (last ? (zz == 0 && b >= need) : pos >= e0) break;
            if (pos >= e0 && last) { bad = true; break; }               // the interval's data ended early
            if (zz == 0) ++b;
            const bool in_range = b >= 1 && b <= need;
            if (!in_range) { bad = true; break; }
            bad |= !decode_symbol(us, s_dc, s_ac, L, pos, blk, zz, coef + (iv_blk0 + b - 1) * 64);
        }
        if (last && !bad && pos + 8 <= e0) bad = true;                  // more than the padding left
        if (bad) s_bad = 1;
    }
    __syncthreads();
    if (s_bad) {
        for (int64_t i = tid; i < nblocks * 8; i += kThreads) reinterpret_cast<int4*>(coef)[i] = make_int4(0, 0, 0, 0);
        if (tid == 0) B.status[blockIdx.x] = 2;
        return;
    }
    // ---- 7. DC: segmented prefix sum of the differences per component in decode order, restarting at every interval
    for (int c = 0; c < 3; ++c) {
        const int per = im.bpm == 6 && c == 0 ? 4 : 1;                 // blocks of component c per MCU
        const int first = c == 0 ? 0 : (im.bpm == 6 ? 3 + c : c);
        const int64_t ne = (int64_t)mcus * per;
        const int chunk = (int)((ne + kThreads - 1) / kThreads);
        const int64_t e0 = min(ne, (int64_t)tid * chunk), e1 = min(ne, e0 + chunk);
        auto gidx = [&](int64_t e) { return (e / per) * im.bpm + first + e % per; };
        auto reset = [&](int64_t e) { return e % per == 0 && (e / per) % im.ri == 0; };
        int f = 0, v = 0;
        for (int64_t e = e0; e < e1; ++e) {
            const int d = coef[gidx(e) * 64];
            if (reset(e)) { f = 1; v = d; } else v += d;
        }
        int cf;
        int acc = block_seg_scan(f, v, sh, sh2, cf);
        for (int64_t e = e0; e < e1; ++e) {
            int16_t* p = coef + gidx(e) * 64;
            acc = reset(e) ? *p : acc + *p;
            *p = (int16_t)acc;
        }
        __syncthreads();
    }
    if (tid == 0) B.status[blockIdx.x] = 0;
}

// ---- jidctint.c, one 8x8 block per 8 threads: thread t does column t (pass 1), then row t (pass 2)
constexpr int F0_298 = 2446, F0_390 = 3196, F0_541 = 4433, F0_765 = 6270, F0_899 = 7373, F1_175 = 9633, F1_501 = 12299,
              F1_847 = 15137, F1_961 = 16069, F2_053 = 16819, F2_562 = 20995, F3_072 = 25172;

__device__ __forceinline__ void idct8(int d0, int d1, int d2, int d3, int d4, int d5, int d6, int d7, int (&o)[8])
{
    int z1 = (d2 + d6) * F0_541;
    const int tmp2 = z1 + d6 * -F1_847, tmp3 = z1 + d2 * F0_765;
    const int tmp0 = (d0 + d4) << 13, tmp1 = (d0 - d4) << 13;
    const int tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
    int t0 = d7, t1 = d5, t2 = d3, t3 = d1;
    z1 = t0 + t3;
    int z2 = t1 + t2, z3 = t0 + t2, z4 = t1 + t3;
    const int z5 = (z3 + z4) * F1_175;
    t0 *= F0_298; t1 *= F2_053; t2 *= F3_072; t3 *= F1_501;
    z1 *= -F0_899; z2 *= -F2_562; z3 *= -F1_961; z4 *= -F0_390;
    z3 += z5; z4 += z5;
    t0 += z1 + z3; t1 += z2 + z4; t2 += z2 + z3; t3 += z1 + z4;
    o[0] = tmp10 + t3; o[7] = tmp10 - t3; o[1] = tmp11 + t2; o[6] = tmp11 - t2;
    o[2] = tmp12 + t1; o[5] = tmp12 - t1; o[3] = tmp13 + t0; o[4] = tmp13 - t0;
}

// libjpeg's post-IDCT range limit: index x & 1023 of prepare_range_limit_table's table
__device__ __forceinline__ uint8_t range_limit(int x)
{
    const int i = x & 1023;
    return (uint8_t)(i < 128 ? i + 128 : i < 512 ? 255 : i < 896 ? 0 : i - 896);
}

constexpr int kIdctBlocks = 32;         // 8x8 blocks per 256-thread CTA

__global__ void __launch_bounds__(256) jpeg_idct_kernel(Bufs B)
{
    const JpegImage& im = B.img[blockIdx.y];
    const int64_t nblocks = (int64_t)im.mcux * im.mcuy * im.bpm;
    const int lb = threadIdx.x >> 3, t = threadIdx.x & 7;
    const int64_t g = (int64_t)blockIdx.x * kIdctBlocks + lb;
    __shared__ int ws[kIdctBlocks][8][9];
    const bool live = g < nblocks;
    int c = 0, by = 0, bx = 0;
    if (live) {
        const int64_t m = g / im.bpm;
        const int b = (int)(g % im.bpm);
        const int my = (int)(m / im.mcux), mx = (int)(m % im.mcux);
        if (im.bpm == 6 && b < 4) { by = 2 * my + (b >> 1); bx = 2 * mx + (b & 1); }
        else { c = im.bpm == 6 ? b - 3 : b; by = my; bx = mx; }
        const int16_t* in = B.coef + (im.coef_off + g) * 64;
        const uint16_t* q = im.q[c];
        int d[8];
        bool ac0 = true;
        for (int r = 0; r < 8; ++r) {
            d[r] = (int)in[r * 8 + t] * (int)q[r * 8 + t];
            ac0 = ac0 && (r == 0 || d[r] == 0);
        }
        if (ac0) {
            for (int r = 0; r < 8; ++r) ws[lb][r][t] = d[0] << 2;
        } else {
            int o[8];
            idct8(d[0], d[1], d[2], d[3], d[4], d[5], d[6], d[7], o);
            for (int r = 0; r < 8; ++r) ws[lb][r][t] = (o[r] + (1 << 10)) >> 11;
        }
    }
    __syncthreads();
    if (!live) return;
    const int* w = ws[lb][t];
    uint8_t px[8];
    if (w[1] == 0 && w[2] == 0 && w[3] == 0 && w[4] == 0 && w[5] == 0 && w[6] == 0 && w[7] == 0) {
        const uint8_t v = range_limit((w[0] + 16) >> 5);
        for (int k = 0; k < 8; ++k) px[k] = v;
    } else {
        int o[8];
        idct8(w[0], w[1], w[2], w[3], w[4], w[5], w[6], w[7], o);
        for (int k = 0; k < 8; ++k) px[k] = range_limit((o[k] + (1 << 17)) >> 18);
    }
    const int s = c == 0 ? im.sub : 1;
    const int64_t pitch = (int64_t)im.mcux * 8 * s;
    uint8_t* dst = B.planes + im.plane_off[c] + (int64_t)(by * 8 + t) * pitch + bx * 8;
    uint2 v;
    v.x = px[0] | px[1] << 8 | px[2] << 16 | (uint32_t)px[3] << 24;
    v.y = px[4] | px[5] << 8 | px[6] << 16 | (uint32_t)px[7] << 24;
    *reinterpret_cast<uint2*>(dst) = v;
}

// ---- h2v2 fancy upsampling (jdsample.c) + YCbCr -> BGR (jdcolor.c, SCALEBITS 16), one thread per output pixel
constexpr int fix16(double x) { return (int)(x * 65536.0 + 0.5); }

__device__ __forceinline__ int chroma(const uint8_t* p, int64_t pitch, int sub, int dh, int dw, int y, int x)
{
    if (sub == 1) return p[(int64_t)y * pitch + x];
    const int cy = y >> 1, cx = x >> 1;
    if (dw <= 2) return p[(int64_t)cy * pitch + cx];                  // h2v2_upsample: replication
    const int oy = (y & 1) ? min(cy + 1, dh - 1) : max(cy - 1, 0);
    const uint8_t* r0 = p + (int64_t)cy * pitch;
    const uint8_t* r1 = p + (int64_t)oy * pitch;
    const int s = 3 * r0[cx] + r1[cx];
    const int nx = (x & 1) ? min(cx + 1, dw - 1) : max(cx - 1, 0);
    const int sn = 3 * r0[nx] + r1[nx];
    return (x & 1) ? (3 * s + sn + 7) >> 4 : (3 * s + sn + 8) >> 4;
}

__global__ void __launch_bounds__(256) jpeg_color_kernel(Bufs B)
{
    const JpegImage& im = B.img[blockIdx.y];
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (int64_t)im.h * im.w) return;
    const int y = (int)(i / im.w), x = (int)(i % im.w);
    const int64_t ypitch = (int64_t)im.mcux * 8 * im.sub, cpitch = (int64_t)im.mcux * 8;
    const int Y = B.planes[im.plane_off[0] + (int64_t)y * ypitch + x];
    const int dh = (im.h + im.sub - 1) / im.sub, dw = (im.w + im.sub - 1) / im.sub;
    const int cb = chroma(B.planes + im.plane_off[1], cpitch, im.sub, dh, dw, y, x) - 128;
    const int cr = chroma(B.planes + im.plane_off[2], cpitch, im.sub, dh, dw, y, x) - 128;
    const int r = Y + ((fix16(1.40200) * cr + 32768) >> 16);
    const int g = Y + ((-fix16(0.34414) * cb + 32768 - fix16(0.71414) * cr) >> 16);
    const int b = Y + ((fix16(1.77200) * cb + 32768) >> 16);
    uint8_t* o = B.out + im.out_off + i * 3;
    o[0] = (uint8_t)min(max(b, 0), 255);
    o[1] = (uint8_t)min(max(g, 0), 255);
    o[2] = (uint8_t)min(max(r, 0), 255);
}

}  // namespace
}  // namespace occ

using namespace occ;

struct occb200_jpeg {
    std::vector<Prepared> imgs;
    int64_t in_bytes = 0, unst_bytes = 0, n_iv = 0, n_sub = 0, n_coef = 0, plane_bytes = 0, out_bytes = 0;
    int64_t max_pixels = 0, max_blocks = 0;
    uint8_t* pinned = nullptr;
    size_t pinned_bytes = 0;
    int32_t* status_pinned = nullptr;
    cudaEvent_t staged = nullptr;       // the last upload has left `pinned`
    bool staged_recorded = false;
    DevBuf in, unst, iv, sub_first, sub_iv, cnt, st, ex, nst, coef, planes, status;
};

namespace occ {

int jpeg_prepare(occb200_jpeg* d, int n, const void* const* data, const int64_t* size, int want_h, int want_w)
{
    OCC_CHECK(d && n >= 1 && data && size, "jpeg: null pointer or no image");
    d->imgs.resize(n);
    int64_t in_b = ((int64_t)n * sizeof(JpegImage) + 255) & ~(int64_t)255, un_b = 0, iv_n = 0, sub_n = 0, coef_n = 0, pl = 0,
            out_b = 0;
    int64_t maxpx = 0, maxblk = 0;
    for (int i = 0; i < n; ++i) {
        Prepared& p = d->imgs[i];
        if (parse_jpeg(static_cast<const uint8_t*>(data[i]), size[i], p)) {
            set_last_error("jpeg image " + std::to_string(i) + ": " + occb200_last_error());
            return 1;
        }
        JpegImage& im = p.im;
        OCC_CHECK(want_h <= 0 || (im.h == want_h && im.w == want_w),
                  "jpeg image " + std::to_string(i) + " is " + std::to_string(im.w) + "x" + std::to_string(im.h) +
                      " (w x h), the frame format is " + std::to_string(want_w) + "x" + std::to_string(want_h));
        im.seg_off = un_b;
        un_b += (im.seg_len + kPad + 15) & ~15;
        im.iv_off = iv_n;
        iv_n += im.n_iv + 1;
        im.sub_off = sub_n;
        sub_n += im.n_sub_cap;
        im.coef_off = coef_n;
        const int64_t nb = (int64_t)im.mcux * im.mcuy * im.bpm;
        coef_n += nb;
        const int64_t cw = (int64_t)im.mcux * 8, ch = (int64_t)im.mcuy * 8;
        im.plane_off[0] = pl;
        pl += cw * ch * im.sub * im.sub;
        im.plane_off[1] = pl;
        pl += cw * ch;
        im.plane_off[2] = pl;
        pl += cw * ch;
        pl = (pl + 15) & ~(int64_t)15;
        im.out_off = out_b;
        out_b += (int64_t)im.h * im.w * 3;
        maxpx = std::max(maxpx, (int64_t)im.h * im.w);
        maxblk = std::max(maxblk, nb);
    }
    d->in_bytes = in_b + un_b;
    d->unst_bytes = un_b;
    d->n_iv = iv_n;
    d->n_sub = sub_n;
    d->n_coef = coef_n;
    d->plane_bytes = pl;
    d->out_bytes = out_b;
    d->max_pixels = maxpx;
    d->max_blocks = maxblk;
    return 0;
}

int64_t jpeg_out_bytes(const occb200_jpeg* d) { return d->out_bytes; }

int jpeg_upload(occb200_jpeg* d, cudaStream_t copy, cudaStream_t st)
{
    const int n = (int)d->imgs.size();
    if (!d->staged) OCC_CUDA(cudaEventCreateWithFlags(&d->staged, cudaEventDisableTiming));
    if (d->staged_recorded) OCC_CUDA(cudaEventSynchronize(d->staged));     // the previous upload has left the staging buffer
    if (d->pinned_bytes < (size_t)d->in_bytes) {
        if (d->pinned) OCC_CUDA(cudaFreeHost(d->pinned));
        d->pinned = nullptr;
        d->pinned_bytes = 0;
        OCC_CUDA(cudaMallocHost(&d->pinned, d->in_bytes));
        d->pinned_bytes = d->in_bytes;
    }
    const int64_t hdr = d->in_bytes - d->unst_bytes;
    for (int i = 0; i < n; ++i) {
        memcpy(d->pinned + i * sizeof(JpegImage), &d->imgs[i].im, sizeof(JpegImage));
        memcpy(d->pinned + hdr + d->imgs[i].im.seg_off, d->imgs[i].seg, d->imgs[i].im.seg_len);
    }
    if (d->in.bytes < (size_t)d->in_bytes && d->in.alloc(d->in_bytes)) return 2;
    OCC_CUDA(cudaMemcpyAsync(d->in.p, d->pinned, d->in_bytes, cudaMemcpyHostToDevice, copy));
    OCC_CUDA(cudaEventRecord(d->staged, copy));
    d->staged_recorded = true;
    if (copy != st) OCC_CUDA(cudaStreamWaitEvent(st, d->staged, 0));
    return 0;
}

// grow-only device buffers, so that a frame's scratch stays allocated from frame to frame
int grow(DevBuf& b, size_t n) { return b.bytes < n && b.alloc(n) ? 2 : 0; }

int jpeg_decode(occb200_jpeg* d, uint8_t* out, cudaStream_t st)
{
    const int n = (int)d->imgs.size();
    if (grow(d->unst, d->unst_bytes) || grow(d->iv, d->n_iv * 4) || grow(d->sub_first, d->n_iv * 4) ||
        grow(d->sub_iv, d->n_sub * 4) || grow(d->cnt, d->n_sub * 4) || grow(d->st, d->n_sub * 8) || grow(d->ex, d->n_sub * 8) ||
        grow(d->nst, d->n_sub * 8) || grow(d->coef, d->n_coef * 128) || grow(d->planes, d->plane_bytes) ||
        grow(d->status, (size_t)n * 4))
        return 2;
    if (!d->status_pinned) OCC_CUDA(cudaMallocHost(&d->status_pinned, 64 * 4));
    Bufs B;
    B.img = d->in.as<JpegImage>();
    B.in = d->in.as<uint8_t>() + (d->in_bytes - d->unst_bytes);
    B.unst = d->unst.as<uint8_t>();
    B.iv = d->iv.as<int32_t>();
    B.sub_first = d->sub_first.as<int32_t>();
    B.sub_iv = d->sub_iv.as<int32_t>();
    B.cnt = d->cnt.as<int32_t>();
    B.st = d->st.as<uint2>();
    B.ex = d->ex.as<uint2>();
    B.nst = d->nst.as<uint2>();
    B.coef = d->coef.as<int16_t>();
    B.planes = d->planes.as<uint8_t>();
    B.out = out;
    B.status = d->status.as<int32_t>();
    jpeg_entropy_kernel<<<n, kThreads, 0, st>>>(B);
    OCC_CUDA(cudaGetLastError());
    jpeg_idct_kernel<<<dim3(ceil_div(d->max_blocks, kIdctBlocks), n), 256, 0, st>>>(B);
    OCC_CUDA(cudaGetLastError());
    jpeg_color_kernel<<<dim3(ceil_div(d->max_pixels, 256), n), 256, 0, st>>>(B);
    OCC_CUDA(cudaGetLastError());
    OCC_CUDA(cudaMemcpyAsync(d->status_pinned, d->status.p, (size_t)std::min(n, 64) * 4, cudaMemcpyDeviceToHost, st));
    return 0;
}

int jpeg_status_host(const occb200_jpeg* d)
{
    int s = 0;
    for (int i = 0; i < std::min((int)d->imgs.size(), 64); ++i)
        if (d->status_pinned[i]) s |= 1 << (i & 31);
    return s;
}

}  // namespace occ

extern "C" {

int occb200_jpeg_create(occb200_jpeg** out)
{
    OCC_CHECK(out, "null pointer");
    *out = new occb200_jpeg();
    return 0;
}

void occb200_jpeg_destroy(occb200_jpeg* d)
{
    if (!d) return;
    if (d->staged) {
        cudaEventSynchronize(d->staged);
        cudaEventDestroy(d->staged);
    }
    if (d->pinned) cudaFreeHost(d->pinned);
    if (d->status_pinned) cudaFreeHost(d->status_pinned);
    delete d;
}

int occb200_jpeg_info(const void* data, int64_t size, int* h, int* w)
{
    OCC_CHECK(data && h && w, "null pointer");
    Prepared p;
    if (parse_jpeg(static_cast<const uint8_t*>(data), size, p)) return 1;
    *h = p.im.h;
    *w = p.im.w;
    return 0;
}

int occb200_jpeg_decode(occb200_jpeg* d, int n, const void* const* data, const int64_t* sizes, uint8_t* out, int64_t out_bytes,
                        void* stream)
{
    OCC_CHECK(d && out, "null pointer");
    if (jpeg_prepare(d, n, data, sizes, 0, 0)) return 1;
    OCC_CHECK(out_bytes == d->out_bytes, "jpeg: output holds " + std::to_string(out_bytes) + " bytes, the images need " +
                                             std::to_string(d->out_bytes));
    cudaStream_t st = (cudaStream_t)stream;
    if (jpeg_upload(d, st, st)) return 2;
    return jpeg_decode(d, out, st);
}

int occb200_jpeg_status(occb200_jpeg* d, int* status)
{
    OCC_CHECK(d && status, "null pointer");
    OCC_CHECK(d->status_pinned != nullptr, "jpeg: no decode has run");
    *status = jpeg_status_host(d);
    return 0;
}

}  // extern "C"
