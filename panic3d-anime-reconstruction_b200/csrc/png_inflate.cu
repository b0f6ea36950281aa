// Device PNG decoder (the input-side partner of png_deflate.cu): N zlib streams (each file's IDAT payloads, concatenated)
// -> N float32 images (N, C, out_h, out_w) in device memory, the tensors `I(path).resize(size)[.convert('RGBA').bg('w')
// .convert('RGB')].t()` gives on the host.
//
// Three kernels, one launch sequence, no host round trip:
//   k_png_inflate    one warp per image.  Lane 0 walks the bit stream (zlib header, stored / fixed / dynamic blocks,
//                    Adler-32 trailer) with table-driven Huffman decoding out of shared memory and writes literals; the
//                    warp copies every match and stored block together, reading the last 32 KB of output from a
//                    window ring in shared memory and writing both the ring and the image's workspace.  Then the
//                    warp sums the Adler-32 of what it wrote and checks it against the trailer.
//   k_png_unfilter   one warp per image, 32 rows at a time: lane k undoes the filter of row r0 + k one pixel behind lane
//                    k - 1 and receives the row above from it by shuffle (Average and Paeth are serial along a row and
//                    each row needs the one above).  Lanes 0 and 1 also tabulate PIL's nearest-neighbour source columns
//                    and rows for the output size.
//   k_png_resample   one thread per output pixel: PIL's nearest resize, 16-bit samples reduced to their high byte, the
//                    optional integer `Image.alpha_composite` onto opaque white, and / 255 into the (N, C, H, W) output.
// Every read and write of an image stays inside its own input span and workspace span; a malformed stream ends with a
// per-image status code (P3D_PNG_E* in p3d_imageio.h), and the other images of the batch decode as if alone.  The bit
// reader and the Huffman decoder are __host__ __device__: p3d_png_inflate_host runs the same decoder on the CPU.
// DESIGN.md 4.7 has the layout, the envelope and the register table.
#include <zlib.h>
#include <string.h>

#include "p3d_common.cuh"
#include "../../include/p3d_imageio.h"

#define P3D_HD __host__ __device__

namespace p3d {
namespace {

constexpr uint64_t kMaxRaw = (uint64_t)1 << 28;   // decompressed bytes per image: h * (1 + w * bytes per pixel)
constexpr int kMaxImages = 65535;
constexpr int kMaxOut = 32768;                    // output side
constexpr int kLitFast = 10, kDistFast = 8;       // first-level table bits; longer codes take the canonical walk
constexpr uint32_t kAdlerMod = 65521;
constexpr int kWin = 32768;                       // deflate window

__constant__ uint16_t c_lbase[29] = {3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115,
                                     131, 163, 195, 227, 258};
__constant__ uint8_t c_lext[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
__constant__ uint16_t c_dbase[30] = {1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537,
                                     2049, 3073, 4097, 6145, 8193, 12289, 16385, 24577};
__constant__ uint8_t c_dext[30] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13};
__constant__ uint8_t c_clorder[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
#ifndef __CUDA_ARCH__
static const uint16_t h_lbase[29] = {3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115,
                                     131, 163, 195, 227, 258};
static const uint8_t h_lext[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
static const uint16_t h_dbase[30] = {1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537,
                                     2049, 3073, 4097, 6145, 8193, 12289, 16385, 24577};
static const uint8_t h_dext[30] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13};
static const uint8_t h_clorder[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
#endif

#ifdef __CUDA_ARCH__
#define P3D_TAB(name) c_##name
#else
#define P3D_TAB(name) h_##name
#endif

// ---------------------------------------------------------------- the envelope (shared by the queries and the kernels)
P3D_HD inline bool supported(int channels, int depth) {
    return (channels == 1 && depth == 8) || ((channels == 3 || channels == 4) && (depth == 8 || depth == 16));
}
// decompressed bytes of one image, 0 outside the envelope (each factor bounded before it is multiplied)
P3D_HD inline uint64_t raw_bytes(int h, int w, int channels, int depth) {
    if (h < 1 || w < 1 || !supported(channels, depth)) return 0;
    const uint64_t bpp = (uint64_t)channels * (depth / 8);
    if ((uint64_t)w > (kMaxRaw - 1) / bpp) return 0;
    const uint64_t row = 1 + (uint64_t)w * bpp;
    if ((uint64_t)h > kMaxRaw / row) return 0;
    return (uint64_t)h * row;
}
P3D_HD inline uint64_t align16(uint64_t x) { return (x + 15) & ~(uint64_t)15; }
// workspace of one image: its decompressed bytes, then the int32 source columns (out_w) and rows (out_h)
P3D_HD inline uint64_t ws_bytes(int h, int w, int channels, int depth, int out_h, int out_w) {
    const uint64_t raw = raw_bytes(h, w, channels, depth);
    if (!raw || out_h < 1 || out_w < 1 || out_h > kMaxOut || out_w > kMaxOut) return 0;
    return align16(raw) + align16(4 * ((uint64_t)out_h + out_w));
}

struct Batch {
    const uint8_t* in;
    uint64_t in_bytes;
    const p3d_png_decode_job* jobs;
    uint8_t* ws;
    uint64_t ws_bytes;
    float* out;
    int32_t* status;
    int n, out_h, out_w, out_c, white;
};

// 0 if job i lies inside the buffers and the envelope, else P3D_PNG_EJOB
P3D_HD inline int check_job(const p3d_png_decode_job& j, const Batch& b) {
    const uint64_t need = ws_bytes(j.h, j.w, j.channels, j.depth, b.out_h, b.out_w);
    if (!need || j.slot < 0 || j.slot >= b.n || (!b.white && j.channels != b.out_c)) return P3D_PNG_EJOB;
    if (j.in_offset > b.in_bytes || j.in_bytes > b.in_bytes - j.in_offset) return P3D_PNG_EJOB;
    if ((j.ws_offset & 15) || j.ws_offset > b.ws_bytes || need > b.ws_bytes - j.ws_offset) return P3D_PNG_EJOB;
    return P3D_PNG_OK;
}

// ---------------------------------------------------------------- bit reader (LSB first, RFC 1951 3.1.1)
struct BitReader {
    const uint8_t* p;
    uint64_t n;        // bytes in the span
    uint64_t pos;      // next byte to load (past n: zeros are loaded)
    uint64_t buf;
    int cnt;           // bits held in buf

    P3D_HD void refill() {   // to at least 57 bits; independent loads
        const int k = (63 - cnt) >> 3;
#pragma unroll
        for (int i = 0; i < 8; ++i)
            if (i < k) {
                const uint64_t q = pos + i;
                buf |= (uint64_t)(q < n ? p[q] : 0) << (cnt + 8 * i);
            }
        pos += k;
        cnt += 8 * k;
    }
    P3D_HD uint32_t bits(int k) {   // k <= 32, cnt >= k
        const uint32_t v = (uint32_t)(buf & ((1ull << k) - 1));
        buf >>= k;
        cnt -= k;
        return v;
    }
    P3D_HD bool past_end() const { return pos * 8 - (uint64_t)cnt > n * 8; }   // consumed a bit the span does not have
    P3D_HD uint64_t byte_pos() const { return pos - (uint64_t)(cnt >> 3); }     // after align(): the next unread byte
    P3D_HD void align() { bits(cnt & 7); }
    P3D_HD void seek(uint64_t q) { pos = q; buf = 0; cnt = 0; }
};

// ---------------------------------------------------------------- canonical Huffman codes (RFC 1951 3.2.2)
// count/sym: the canonical form, walked one bit at a time for codes longer than the first-level table (puff's decode);
// fast[]: first-level table, entry = symbol | length << 9 for codes of <= fast_bits bits, 0 = walk.
struct Huff {
    uint16_t count[16];
    uint16_t sym[288];
};

// zlib's inflate_table rules: over-subscribed lengths are refused; an incomplete code only when it is a single code of
// one bit (or no code at all, which fails when used).  Returns false on a refused set.
P3D_HD inline bool build(Huff& h, uint16_t* fast, int fast_bits, const uint8_t* len, int n) {
    for (int l = 0; l < 16; ++l) h.count[l] = 0;
    for (int s = 0; s < n; ++s) h.count[len[s]]++;
    int max = 0;
    for (int l = 1; l < 16; ++l)
        if (h.count[l]) max = l;
    int left = 1;
    for (int l = 1; l < 16; ++l) {
        left = (left << 1) - h.count[l];
        if (left < 0) return false;
    }
    if (left > 0 && max > 1) return false;
    uint16_t offs[16], next[16];
    offs[1] = 0;
    for (int l = 1; l < 15; ++l) offs[l + 1] = offs[l] + h.count[l];
    int code = 0;
    h.count[0] = 0;
    for (int l = 1; l < 16; ++l) { code = (code + h.count[l - 1]) << 1; next[l] = (uint16_t)code; }
    for (int e = 0; e < (1 << fast_bits); ++e) fast[e] = 0;
    for (int s = 0; s < n; ++s) {
        const int l = len[s];
        if (!l) continue;
        h.sym[offs[l]++] = (uint16_t)s;
        const uint32_t c = next[l]++;
        if (l > fast_bits) continue;
        uint32_t r = 0;
        for (int b = 0; b < l; ++b) r |= ((c >> b) & 1) << (l - 1 - b);
        for (uint32_t e = r; e < (1u << fast_bits); e += 1u << l) fast[e] = (uint16_t)(s | l << 9);
    }
    return true;
}

// next symbol, or -1 when the bits are not a code of this set; needs 15 bits in the reader
P3D_HD inline int decode(BitReader& br, const Huff& h, const uint16_t* fast, int fast_bits) {
    const uint16_t e = fast[br.buf & ((1u << fast_bits) - 1)];
    if (e) { br.bits(e >> 9); return e & 511; }
    int code = 0, first = 0, index = 0;
    for (int l = 1; l < 16; ++l) {
        code |= (int)((br.buf >> (l - 1)) & 1);
        const int count = h.count[l];
        if (code - count < first) { br.bits(l); return h.sym[index + (code - first)]; }
        index += count;
        first = (first + count) << 1;
        code <<= 1;
    }
    return -1;
}

struct Tables {
    Huff lit, dist, cl;
    uint16_t lfast[1 << kLitFast], dfast[1 << kDistFast], clfast[1 << 7];
    uint8_t lens[286 + 30];
    int kind;          // what the tables hold: 0 nothing, 1 fixed, 2 a dynamic block
};

// What lane 0 hands to the warp: a match or a stored run to copy, the end of the stream, or an error.
enum { TOK_MATCH = 0, TOK_STORED = 1, TOK_END = 2, TOK_ERROR = 3 };
struct Token {
    int kind;
    uint32_t len;       // bytes to write at dst
    uint64_t dst, src;  // src: match distance, or the stored run's input byte offset
};

// The decoder state of one stream.  run() writes literals itself and returns at each copy, so the copies can be shared.
struct Inflater {
    BitReader br;
    uint64_t out_len, p;  // output size, bytes written
    int state;            // 0: zlib header, 1: block header, 2: inside a Huffman block, 3: trailer
    bool last;
    uint32_t adler;       // from the trailer

    P3D_HD void init(const uint8_t* in, uint64_t n, uint64_t raw) {
        br.p = in; br.n = n; br.pos = 0; br.buf = 0; br.cnt = 0;
        out_len = raw; p = 0; state = 0; last = false; adler = 0;
    }
    P3D_HD Token fail(int code) { Token t; t.kind = TOK_ERROR; t.len = (uint32_t)code; t.dst = t.src = 0; return t; }

    P3D_HD int dynamic_header(Tables& t) {
        br.refill();
        const int hlit = (int)br.bits(5) + 257, hdist = (int)br.bits(5) + 1, hclen = (int)br.bits(4) + 4;
        if (hlit > 286 || hdist > 30) return P3D_PNG_ECODES;
        uint8_t cl[19];
        for (int i = 0; i < 19; ++i) cl[i] = 0;
        for (int i = 0; i < hclen; ++i) {
            if (br.cnt < 3) br.refill();
            cl[P3D_TAB(clorder)[i]] = (uint8_t)br.bits(3);
        }
        if (br.past_end()) return P3D_PNG_ETRUNCATED;
        if (!build(t.cl, t.clfast, 7, cl, 19)) return P3D_PNG_ECODES;
        for (int i = 0; i < hlit + hdist;) {
            br.refill();
            const int s = decode(br, t.cl, t.clfast, 7);
            if (br.past_end()) return P3D_PNG_ETRUNCATED;
            if (s < 0) return P3D_PNG_ECODES;
            if (s < 16) { t.lens[i++] = (uint8_t)s; continue; }
            int rep, v = 0;
            if (s == 16) {
                if (i == 0) return P3D_PNG_ECODES;
                v = t.lens[i - 1];
                rep = 3 + (int)br.bits(2);
            } else {
                rep = s == 17 ? 3 + (int)br.bits(3) : 11 + (int)br.bits(7);
            }
            if (br.past_end()) return P3D_PNG_ETRUNCATED;
            if (i + rep > hlit + hdist) return P3D_PNG_ECODES;
            while (rep--) t.lens[i++] = (uint8_t)v;
        }
        if (t.lens[256] == 0) return P3D_PNG_ECODES;                       // no end-of-block code
        if (!build(t.lit, t.lfast, kLitFast, t.lens, hlit)) return P3D_PNG_ECODES;
        if (!build(t.dist, t.dfast, kDistFast, t.lens + hlit, hdist)) return P3D_PNG_ECODES;
        t.kind = 2;
        return P3D_PNG_OK;
    }

    P3D_HD void fixed_tables(Tables& t) {
        uint8_t l[288];
        for (int i = 0; i < 288; ++i) l[i] = i < 144 ? 8 : i < 256 ? 9 : i < 280 ? 7 : 8;
        build(t.lit, t.lfast, kLitFast, l, 288);
        for (int i = 0; i < 32; ++i) l[i] = 5;                              // 30 and 31 decode, and are refused
        build(t.dist, t.dfast, kDistFast, l, 32);
        t.kind = 1;
    }

    // Decode until the warp has something to copy.  `raw` is this image's output and win[x & mask] its last bytes (the
    // device keeps the 32 KB window in shared memory; the host passes raw itself); only lane 0 calls this.
    P3D_HD Token run(uint8_t* raw, uint8_t* win, uint32_t mask, Tables& t) {
        for (;;) {
            if (state == 0) {
                br.refill();
                const uint32_t cmf = br.bits(8), flg = br.bits(8);
                if (br.past_end()) return fail(P3D_PNG_ETRUNCATED);
                if ((cmf & 15) != 8 || (cmf >> 4) > 7 || (cmf * 256 + flg) % 31 || (flg & 32)) return fail(P3D_PNG_EHEADER);
                state = 1;
            }
            if (state == 3) {
                br.align();
                br.refill();
                uint32_t a = 0;
                for (int i = 0; i < 4; ++i) a = a << 8 | br.bits(8);
                if (br.past_end()) return fail(P3D_PNG_ETRUNCATED);
                if (p != out_len) return fail(P3D_PNG_ESHORT);
                adler = a;
                Token e; e.kind = TOK_END; e.len = 0; e.dst = e.src = 0;
                return e;
            }
            if (state == 1) {
                if (last) { state = 3; continue; }
                br.refill();
                last = br.bits(1);
                const int type = (int)br.bits(2);
                if (br.past_end()) return fail(P3D_PNG_ETRUNCATED);
                if (type == 0) {
                    br.align();
                    br.refill();
                    const uint32_t len = br.bits(16), nlen = br.bits(16);
                    if (br.past_end()) return fail(P3D_PNG_ETRUNCATED);
                    if ((len ^ 0xffffu) != nlen) return fail(P3D_PNG_EBLOCK);
                    const uint64_t q = br.byte_pos();
                    if (len > br.n - q) return fail(P3D_PNG_ETRUNCATED);
                    if (len > out_len - p) return fail(P3D_PNG_ELONG);
                    br.seek(q + len);
                    if (!len) continue;                                     // a sync flush
                    Token s; s.kind = TOK_STORED; s.len = len; s.dst = p; s.src = q;
                    p += len;
                    return s;
                }
                if (type == 3) return fail(P3D_PNG_EBLOCK);
                if (type == 1) {
                    if (t.kind != 1) fixed_tables(t);
                } else {
                    t.kind = 0;
                    const int e = dynamic_header(t);
                    if (e) return fail(e);
                }
                state = 2;
            }
            // state 2: literals are written here; a match goes to the warp
            for (;;) {
                br.refill();
                const int s = decode(br, t.lit, t.lfast, kLitFast);
                if (br.past_end()) return fail(P3D_PNG_ETRUNCATED);
                if (s < 0) return fail(P3D_PNG_ESYMBOL);
                if (s < 256) {
                    if (p >= out_len) return fail(P3D_PNG_ELONG);
                    raw[p] = (uint8_t)s;
                    win[(uint32_t)p & mask] = (uint8_t)s;
                    ++p;
                    continue;
                }
                if (s == 256) { state = 1; break; }
                if (s > 285) return fail(P3D_PNG_ESYMBOL);
                const uint32_t len = P3D_TAB(lbase)[s - 257] + br.bits(P3D_TAB(lext)[s - 257]);
                const int ds = decode(br, t.dist, t.dfast, kDistFast);
                if (br.past_end()) return fail(P3D_PNG_ETRUNCATED);
                if (ds < 0 || ds > 29) return fail(P3D_PNG_ESYMBOL);
                const uint32_t dist = P3D_TAB(dbase)[ds] + br.bits(P3D_TAB(dext)[ds]);
                if (br.past_end()) return fail(P3D_PNG_ETRUNCATED);
                if (dist > p) return fail(P3D_PNG_EDISTANCE);
                if (len > out_len - p) return fail(P3D_PNG_ELONG);
                Token m; m.kind = TOK_MATCH; m.len = len; m.dst = p; m.src = dist;
                p += len;
                return m;
            }
        }
    }
};

// byte j of a match: an overlapping copy (distance below the length) repeats the `dist` bytes before it, so every byte
// depends only on bytes written before the match and the warp may write them in any order
P3D_HD inline uint64_t match_src(const Token& m, uint32_t j) { return m.dst - m.src + (m.src >= m.len ? j : j % (uint32_t)m.src); }

// Adler-32 sums of raw[0, n) with byte i weighted by n - i (RFC 1950 8.2: b = n + sum (n - i) x_i)
P3D_HD inline uint32_t adler_of(uint64_t n, uint64_t s1, uint64_t s2) {
    return (uint32_t)(((n + s2) % kAdlerMod) << 16 | ((1 + s1) % kAdlerMod));
}

// ---------------------------------------------------------------- k_png_inflate
__global__ void __launch_bounds__(32) k_png_inflate(Batch b) {
    __shared__ Tables t;
    __shared__ uint8_t win[kWin];                       // the last 32 KB of output: where matches read
    Inflater st;                                        // lane 0's decoder state, in its registers
    const int lane = threadIdx.x, i = blockIdx.x;
    const p3d_png_decode_job job = b.jobs[i];
    const int jerr = check_job(job, b);
    if (jerr) {
        if (lane == 0) b.status[i] = jerr;
        return;
    }
    const uint8_t* in = b.in + job.in_offset;
    uint8_t* raw = b.ws + job.ws_offset;
    const uint64_t n = raw_bytes(job.h, job.w, job.channels, job.depth);
    if (lane == 0) { st.init(in, job.in_bytes, n); t.kind = 0; }
    Token tk = {TOK_END, 0, 0, 0};
    for (;;) {
        if (lane == 0) tk = st.run(raw, win, kWin - 1, t);
        __syncwarp();                                   // lane 0's literals are visible to the copy
        tk.kind = __shfl_sync(~0u, tk.kind, 0);
        tk.len = __shfl_sync(~0u, tk.len, 0);
        tk.dst = __shfl_sync(~0u, tk.dst, 0);
        tk.src = __shfl_sync(~0u, tk.src, 0);
        if (tk.kind != TOK_MATCH && tk.kind != TOK_STORED) break;
        // In a round every lane reads before any lane writes.  A window slot read in a later round than it is written
        // in would need a distance above 32768 - (length - 1) with the reader behind the writer, which cannot happen:
        // the byte that overwrites slot (dst - dist + j) is byte j + 32768 - dist >= j of the match.
        for (uint32_t j0 = 0; j0 < tk.len; j0 += 32) {
            const uint32_t j = j0 + lane;
            uint8_t v = 0;
            if (j < tk.len) v = tk.kind == TOK_MATCH ? win[(uint32_t)match_src(tk, j) & (kWin - 1)] : in[tk.src + j];
            __syncwarp();
            if (j < tk.len) { win[(uint32_t)(tk.dst + j) & (kWin - 1)] = v; raw[tk.dst + j] = v; }
            __syncwarp();
        }
    }
    int code = tk.kind == TOK_ERROR ? (int)tk.len : P3D_PNG_OK;
    if (code == P3D_PNG_OK) {                          // the Adler-32 of the whole output, by the warp
        uint64_t s1 = 0, s2 = 0;
        const uint32_t* w4 = (const uint32_t*)raw;      // ws_offset is 16-byte aligned
#pragma unroll 4
        for (uint64_t k = lane; k < n / 4; k += 32) {
            const uint32_t v = w4[k];
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                const uint32_t x = (v >> (8 * c)) & 255;
                s1 += x;
                s2 += (n - (4 * k + c)) * x;
            }
        }
        for (uint64_t k = (n / 4) * 4 + lane; k < n; k += 32) { s1 += raw[k]; s2 += (n - k) * raw[k]; }
        s1 %= kAdlerMod;
        s2 %= kAdlerMod;
        for (int o = 16; o; o >>= 1) { s1 += __shfl_xor_sync(~0u, s1, o); s2 += __shfl_xor_sync(~0u, s2, o); }
        if (adler_of(n, s1, s2) != __shfl_sync(~0u, st.adler, 0)) code = P3D_PNG_EADLER;
    }
    if (lane == 0) b.status[i] = code;
}

// ---------------------------------------------------------------- k_png_unfilter
__device__ __forceinline__ int paeth(int a, int bb, int c) {
    const int q = a + bb - c, pa = abs(q - a), pb = abs(q - bb), pc = abs(q - c);
    return pa <= pb && pa <= pc ? a : pb <= pc ? bb : c;
}

// PIL's nearest-neighbour source index of each output index: ImagingScaleAffine's double accumulation, -1 past the edge
__device__ void nearest_table(int32_t* tab, int n_in, int n_out) {
    const double scale = (double)n_in / n_out;
    double x = scale * 0.5;
    for (int o = 0; o < n_out; ++o, x += scale) {
        const int v = x < 0.0 ? -1 : (int)x;
        tab[o] = v < n_in ? v : -1;
    }
}

// rows r0 .. r0 + 31 of one image, lane k on row r0 + k, one pixel (BPP bytes, packed in a u64) per step
template <int BPP>
__device__ void unfilter_rows(uint8_t* raw, int h, int w) {
    const int lane = threadIdx.x;
    const uint64_t stride = 1 + (uint64_t)w * BPP;
    for (int r0 = 0; r0 < h; r0 += 32) {
        const int r = r0 + lane;
        uint8_t* row = raw + (uint64_t)r * stride;
        const int type = r < h ? row[0] : 0;
        uint64_t cur = 0, up = 0;          // this row's pixel x - 1 and the row above's pixel x - 1
        for (int s = 0; s < w + 31; ++s) {
            const int x = s - lane;
            const uint64_t prev = cur;                       // a: left
            const uint64_t ul = up;                          // c: upper left
            uint64_t above = __shfl_up_sync(~0u, cur, 1);    // b: lane k - 1 finished this column of its row last step
            if (lane == 0) {
                above = 0;
                if (r0 > 0 && x >= 0 && x < w) {
                    const uint8_t* q = raw + (uint64_t)(r0 - 1) * stride + 1 + (uint64_t)x * BPP;
#pragma unroll
                    for (int c = 0; c < BPP; ++c) above |= (uint64_t)q[c] << (8 * c);
                }
            }
            if (r < h && x >= 0 && x < w) {
                uint8_t* q = row + 1 + (uint64_t)x * BPP;
                uint64_t v = 0;
#pragma unroll
                for (int c = 0; c < BPP; ++c) {
                    const int a = x ? (int)((prev >> (8 * c)) & 255) : 0;
                    const int bb = (int)((above >> (8 * c)) & 255);
                    const int cc = x ? (int)((ul >> (8 * c)) & 255) : 0;
                    const int pred = type == 0 ? 0 : type == 1 ? a : type == 2 ? bb : type == 3 ? (a + bb) >> 1 : paeth(a, bb, cc);
                    const uint8_t o = (uint8_t)(q[c] + pred);
                    q[c] = o;
                    v |= (uint64_t)o << (8 * c);
                }
                cur = v;
                up = above;
            }
        }
        __syncwarp();                                        // row r0 + 31 is in memory for the next band's lane 0
    }
}

__global__ void __launch_bounds__(32) k_png_unfilter(Batch b) {
    const int lane = threadIdx.x, i = blockIdx.x;
    if (b.status[i] != P3D_PNG_OK) return;
    const p3d_png_decode_job job = b.jobs[i];
    uint8_t* raw = b.ws + job.ws_offset;
    const int bpp = job.channels * (job.depth / 8);
    const uint64_t stride = 1 + (uint64_t)job.w * bpp;
    bool bad = false;
    for (int r = lane; r < job.h; r += 32) bad |= raw[(uint64_t)r * stride] > 4;
    if (__any_sync(~0u, bad)) {
        if (lane == 0) b.status[i] = P3D_PNG_EFILTER;
        return;
    }
    int32_t* tab = (int32_t*)(raw + align16(raw_bytes(job.h, job.w, job.channels, job.depth)));
    if (lane == 0) nearest_table(tab, job.w, b.out_w);
    if (lane == 1) nearest_table(tab + b.out_w, job.h, b.out_h);
    __syncwarp();
    switch (bpp) {
        case 1: unfilter_rows<1>(raw, job.h, job.w); break;
        case 3: unfilter_rows<3>(raw, job.h, job.w); break;
        case 4: unfilter_rows<4>(raw, job.h, job.w); break;
        case 6: unfilter_rows<6>(raw, job.h, job.w); break;
        default: unfilter_rows<8>(raw, job.h, job.w); break;
    }
}

// ---------------------------------------------------------------- k_png_resample
// PIL's Image.alpha_composite of (v, a) over opaque white (libImaging/AlphaComposite.c, 7 bits of precision)
__device__ __forceinline__ uint32_t over_white(uint32_t v, uint32_t a) {
    if (a == 0) return 255;
    const uint32_t outa255 = a * 255 + 255 * (255 - a);
    const uint32_t coef1 = a * 255 * 255 * 128 / outa255, coef2 = 255 * 128 - coef1;
    const uint32_t tmp = v * coef1 + 255 * coef2 + (0x80 << 7);
    return (((tmp >> 8) + tmp) >> 8) >> 7;
}

__global__ void __launch_bounds__(256) k_png_resample(Batch b) {
    const int i = blockIdx.y;
    const uint64_t hw = (uint64_t)b.out_h * b.out_w, o = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (o >= hw) return;
    const p3d_png_decode_job job = b.jobs[i];
    if (job.slot < 0 || job.slot >= b.n) return;        // a refused job: nowhere to write
    float* dst = b.out + (uint64_t)job.slot * b.out_c * hw + o;
    if (b.status[i] != P3D_PNG_OK) {
        for (int c = 0; c < b.out_c; ++c) dst[c * hw] = 0.f;
        return;
    }
    const uint8_t* raw = b.ws + job.ws_offset;
    const int32_t* tab = (const int32_t*)(raw + align16(raw_bytes(job.h, job.w, job.channels, job.depth)));
    const int oy = (int)(o / b.out_w), ox = (int)(o % b.out_w);
    const int sx = tab[ox], sy = tab[b.out_w + oy];
    const int bs = job.depth / 8, bpp = job.channels * bs;
    uint32_t px[4] = {0, 0, 0, 0};                      // outside the source: PIL's zero fill
    if (sx >= 0 && sy >= 0) {
        const uint8_t* q = raw + (uint64_t)sy * (1 + (uint64_t)job.w * bpp) + 1 + (uint64_t)sx * bpp;
#pragma unroll
        for (int c = 0; c < 4; ++c)
            if (c < job.channels) px[c] = q[c * bs];    // 16 bits: the high byte
    }
    if (!b.white) {
#pragma unroll
        for (int c = 0; c < 4; ++c)
            if (c < b.out_c) dst[c * hw] = (float)px[c] / 255.f;
        return;
    }
    if (job.channels == 1) px[1] = px[2] = px[0];       // L -> RGBA: opaque grey
#pragma unroll
    for (int c = 0; c < 3; ++c) dst[c * hw] = (float)(job.channels == 4 ? over_white(px[c], px[3]) : px[c]) / 255.f;
}

// ---------------------------------------------------------------- host inspection
uint32_t be32(const uint8_t* p) { return (uint32_t)p[0] << 24 | (uint32_t)p[1] << 16 | (uint32_t)p[2] << 8 | p[3]; }

}  // namespace
}  // namespace p3d

using namespace p3d;

extern "C" int p3d_png_inspect(const uint8_t* file, size_t len, p3d_png_info* info, uint8_t* stream) {
    P3D_REQUIRE(file && info, "p3d_png_inspect: NULL pointer");
    static const uint8_t sig[8] = {0x89, 'P', 'N', 'G', 0x0d, 0x0a, 0x1a, 0x0a};
    P3D_REQUIRE(len >= 8 && !memcmp(file, sig, 8), "p3d_png_inspect: not a PNG file (signature)");
    memset(info, 0, sizeof(*info));
    size_t o = 8;
    int n_chunks = 0, color = -1;
    bool seen_iend = false, idat_done = false, in_idat = false;
    uint64_t total = 0;
    while (!seen_iend) {
        P3D_REQUIRE(len - o >= 12, "p3d_png_inspect: file ends inside a chunk header at byte %zu (no IEND)", o);
        const uint32_t n = be32(file + o);
        const uint8_t* type = file + o + 4;
        char name[5] = {(char)type[0], (char)type[1], (char)type[2], (char)type[3], 0};
        P3D_REQUIRE(n <= 0x7fffffffu && n <= len - o - 12, "p3d_png_inspect: chunk '%s' at byte %zu: length %u past the end of the file",
                    name, o, n);
        const uint8_t* data = file + o + 8;
        const uint32_t crc = (uint32_t)crc32(crc32(0L, Z_NULL, 0), type, n + 4);
        P3D_REQUIRE(crc == be32(data + n), "p3d_png_inspect: chunk '%s' at byte %zu: CRC mismatch", name, o);
        const bool is_idat = !memcmp(type, "IDAT", 4);
        if (n_chunks == 0)
            P3D_REQUIRE(!memcmp(type, "IHDR", 4) && n == 13, "p3d_png_inspect: the first chunk is '%s', not a 13-byte IHDR", name);
        if (!memcmp(type, "IHDR", 4)) {
            P3D_REQUIRE(n_chunks == 0, "p3d_png_inspect: a second IHDR chunk");
            const uint32_t w = be32(data), h = be32(data + 4);
            const int depth = data[8];
            color = data[9];
            P3D_REQUIRE(w >= 1 && h >= 1 && w <= 0x7fffffffu && h <= 0x7fffffffu, "p3d_png_inspect: IHDR width %u / height %u", w, h);
            P3D_REQUIRE(color == 0 || color == 2 || color == 6,
                        "p3d_png_inspect: IHDR colour type %d is not supported (0 grey, 2 RGB and 6 RGBA are; palette and "
                        "grey+alpha are not)", color);
            P3D_REQUIRE(depth == 8 || (depth == 16 && color != 0),
                        "p3d_png_inspect: IHDR bit depth %d with colour type %d is not supported (8 bits, or 16 for RGB and RGBA)",
                        depth, color);
            P3D_REQUIRE(data[10] == 0, "p3d_png_inspect: IHDR compression method %d", data[10]);
            P3D_REQUIRE(data[11] == 0, "p3d_png_inspect: IHDR filter method %d", data[11]);
            P3D_REQUIRE(data[12] == 0, "p3d_png_inspect: IHDR interlace method %d is not supported (interlaced files)", data[12]);
            info->w = (int32_t)w; info->h = (int32_t)h;
            info->channels = color == 0 ? 1 : color == 2 ? 3 : 4;
            info->depth = depth;
            P3D_REQUIRE(raw_bytes(info->h, info->w, info->channels, info->depth),
                        "p3d_png_inspect: IHDR %u x %u x %d channels at %d bits decompresses past the %llu-byte envelope", w, h,
                        info->channels, depth, (unsigned long long)kMaxRaw);
        } else if (is_idat) {
            P3D_REQUIRE(!idat_done, "p3d_png_inspect: IDAT chunks are not consecutive");
            if (stream && n) memcpy(stream + total, data, n);
            total += n;
            info->n_idat++;
        } else if (!memcmp(type, "IEND", 4)) {
            seen_iend = true;
        } else if (!memcmp(type, "tRNS", 4)) {
            P3D_REQUIRE(color == 6, "p3d_png_inspect: tRNS chunk on colour type %d (a transparent key colour is not supported)",
                        color);
        } else if (!memcmp(type, "PLTE", 4)) {
            P3D_REQUIRE(color != 0, "p3d_png_inspect: PLTE chunk on colour type 0");
        } else {
            P3D_REQUIRE(type[0] & 0x20, "p3d_png_inspect: unknown critical chunk '%s'", name);   // ancillary: skipped
        }
        if (in_idat && !is_idat) idat_done = true;
        in_idat = is_idat;
        o += 12 + (size_t)n;
        ++n_chunks;
    }
    P3D_REQUIRE(info->n_idat > 0, "p3d_png_inspect: no IDAT chunk");
    info->stream_bytes = total;
    return P3D_OK;
}

extern "C" size_t p3d_png_decode_workspace_bytes(int32_t h, int32_t w, int32_t channels, int32_t depth, int32_t out_h,
                                                 int32_t out_w) {
    return (size_t)ws_bytes(h, w, channels, depth, out_h, out_w);
}

extern "C" int p3d_png_inflate_host(const uint8_t* stream, size_t len, uint8_t* raw, size_t raw_len) {
    P3D_REQUIRE((stream || !len) && raw && raw_len >= 1 && raw_len <= kMaxRaw,
                "p3d_png_inflate_host: NULL pointer or raw_len %zu outside 1..%llu", raw_len, (unsigned long long)kMaxRaw);
    Tables* t = new Tables;
    t->kind = 0;
    Inflater st;
    st.init(stream, len, raw_len);
    Token tk;
    for (;;) {
        tk = st.run(raw, raw, ~0u, *t);
        if (tk.kind == TOK_MATCH) {
            for (uint32_t j = 0; j < tk.len; ++j) raw[tk.dst + j] = raw[match_src(tk, j)];
        } else if (tk.kind == TOK_STORED) {
            memcpy(raw + tk.dst, stream + tk.src, tk.len);
        } else {
            break;
        }
    }
    delete t;
    if (tk.kind == TOK_ERROR) return (int)tk.len;
    uint64_t s1 = 0, s2 = 0;
    for (uint64_t k = 0; k < raw_len; ++k) { s1 += raw[k]; s2 += (raw_len - k) * raw[k]; }
    return adler_of(raw_len, s1 % kAdlerMod, s2 % kAdlerMod) == st.adler ? P3D_PNG_OK : P3D_PNG_EADLER;
}

extern "C" int p3d_png_decode_device(const uint8_t* in, size_t in_bytes, const p3d_png_decode_job* jobs, int32_t n,
                                     int32_t out_h, int32_t out_w, int32_t out_channels, int32_t white_background,
                                     void* workspace, size_t workspace_bytes, float* out, int32_t* status, void* stream) {
    P3D_REQUIRE(in && jobs && workspace && out && status, "p3d_png_decode_device: NULL pointer");
    P3D_REQUIRE(n >= 1 && n <= kMaxImages && out_h >= 1 && out_w >= 1 && out_h <= kMaxOut && out_w <= kMaxOut &&
                (white_background ? out_channels == 3 : (out_channels == 1 || out_channels == 3 || out_channels == 4)),
                "p3d_png_decode_device: n=%d out %dx%dx%d (white_background=%d) outside the envelope (1 <= n <= %d, "
                "1 <= out_h, out_w <= %d, 3 channels on white, else 1, 3 or 4)",
                n, out_h, out_w, out_channels, white_background, kMaxImages, kMaxOut);
    Batch b;
    b.in = in; b.in_bytes = in_bytes; b.jobs = jobs; b.ws = (uint8_t*)workspace; b.ws_bytes = workspace_bytes;
    b.out = out; b.status = status; b.n = n; b.out_h = out_h; b.out_w = out_w; b.out_c = out_channels;
    b.white = white_background ? 1 : 0;
    cudaStream_t st = (cudaStream_t)stream;
    k_png_inflate<<<(unsigned)n, 32, 0, st>>>(b);
    P3D_LAUNCH_CHECK();
    k_png_unfilter<<<(unsigned)n, 32, 0, st>>>(b);
    P3D_LAUNCH_CHECK();
    const uint64_t hw = (uint64_t)out_h * out_w;
    k_png_resample<<<dim3((unsigned)((hw + 255) / 256), (unsigned)n), 256, 0, st>>>(b);
    P3D_LAUNCH_CHECK();
    return P3D_OK;
}
