// Device PNG encoder (SURVEY 8f-4): filtered scan-line streams (what k_png_scanlines writes) -> complete PNG files in device
// memory, so the per-view deflate runs on the GPU that rendered the view instead of on rank 0's host threads.
//
// Two kernels, no host round trip:
//   k_deflate_segment  one CTA per (image, 16 KB segment of its stream).  LZ77 over the segment with a 32 KB window that
//                      reaches back into the preceding segments, a greedy parse, per-segment length-limited canonical
//                      Huffman codes, and the smallest of a dynamic, fixed or stored block.  Every non-final segment ends
//                      with a sync flush (an empty stored block), so each segment's bytes start and end on a byte boundary
//                      and the segments concatenate into one deflate stream.  Also its Adler-32 and CRC-32 partials.
//   k_png_assemble     one CTA per image: an exclusive scan of the segment sizes places every segment, the Adler-32 of
//                      the stream and the CRC-32 of IDAT are combined from the partials, and the chunks are written.
// Determinism: the only atomics are max (hash heads), add of integer counts (histograms) and or (bit emission into a
// zeroed buffer); none of their orders shows in the result.  The bytes are a function of the input bytes alone.
// DESIGN.md 4.6 has the layout, the size bound and the register table.
#include "p3d_common.cuh"
#include "../../include/p3d_imageio.h"

namespace p3d {
namespace {

constexpr int kSeg = 16384;                    // input bytes per segment (one CTA)
constexpr int kWin = 32768;                    // deflate window: how far a match may reach back
constexpr int kThreads = 1024;
constexpr int kPer = kSeg / kThreads;          // positions per thread in the per-position passes
constexpr int kHashBits = 13;
constexpr int kSlot = kSeg + 16;               // workspace bytes per segment: stored block + sync flush = kSeg + 10
constexpr int kOutWords = kSlot / 4 + 2;       // emission buffer (one word of slack for the last putbits)
constexpr size_t kMaxStream = (size_t)1 << 28; // per-image stream bytes (16384 segments)
constexpr int kMaxImages = 65535;              // grid.y
constexpr int kHeadBytes = 8 + 25 + 8 + 2;     // signature, IHDR, IDAT length + type, zlib CMF/FLG
constexpr int kTailBytes = 4 + 4 + 12;         // Adler-32, IDAT CRC, IEND
constexpr uint32_t kAdlerMod = 65521;

// dynamic shared memory of k_deflate_segment
constexpr int kOffData = 0;                                   // [window | segment] bytes; the window part later holds the output bits
constexpr int kOffLen = kOffData + kWin + kSeg;               // per position: match length - 3
constexpr int kOffDist = kOffLen + kSeg;                      // per position: match distance (0: none), u16
constexpr int kOffHead = kOffDist + 2 * kSeg;                 // hash heads (position + 1), u32; later the Huffman scratch
constexpr int kOffChosen = kOffHead + 4 * (1 << kHashBits);   // token-start bit per position
constexpr int kSmem = kOffChosen + kSeg / 8;

__constant__ uint16_t c_len_base[29] = {3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99,
                                        115, 131, 163, 195, 227, 258};
__constant__ uint8_t c_len_extra[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
__constant__ uint8_t c_cl_order[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};

struct DeflateArgs {
    const uint8_t* scan;       // n streams of `len` bytes
    uint8_t* slots;            // n * nseg * kSlot
    uint32_t* meta;            // n * nseg * 4: bytes, raw CRC (init 0), Adler sum, Adler weighted sum
    long long len;             // stream bytes per image
    int nseg, bpp, stride;     // bytes per pixel and per scan-line: the match finder's fixed candidate distances
    uint32_t x8[32];           // x^(8 * 2^k) mod the CRC-32 polynomial (reflected), k = 0..31
};

struct AssembleArgs {
    const uint8_t* slots;
    const uint32_t* meta;
    uint8_t* out;
    size_t out_stride;
    uint64_t* out_lens;
    long long len;
    int nseg, h, w, c;
    uint32_t x8[32];
};

// ---------------------------------------------------------------- CRC-32 algebra (zlib's crc32_combine, reflected)
__host__ __device__ inline uint32_t gf2_mul(uint32_t a, uint32_t b) {   // a * b mod P; x^0 is bit 31
    uint32_t p = 0;
    for (int i = 0; i < 32; ++i) {
        if (a & (0x80000000u >> i)) p ^= b;
        b = (b & 1) ? (b >> 1) ^ 0xedb88320u : b >> 1;
    }
    return p;
}
__device__ inline uint32_t x8pow(const uint32_t* x8, unsigned long long m) {   // x^(8 m) mod P
    uint32_t p = 0x80000000u;
    for (int k = 0; m; ++k, m >>= 1)
        if (m & 1) p = gf2_mul(x8[k], p);
    return p;
}
__device__ inline void crc_table(uint32_t* tab) {
    for (int i = threadIdx.x; i < 256; i += blockDim.x) {
        uint32_t c = (uint32_t)i;
        for (int k = 0; k < 8; ++k) c = (c & 1) ? (c >> 1) ^ 0xedb88320u : c >> 1;
        tab[i] = c;
    }
}
__device__ inline uint32_t crc_bytes(const uint32_t* tab, uint32_t c, const uint8_t* p, int n) {
    for (int i = 0; i < n; ++i) c = tab[(c ^ p[i]) & 255] ^ (c >> 8);
    return c;
}

// ---------------------------------------------------------------- block reductions / scan (kThreads threads)
template <class T>
__device__ inline T block_sum(T v, T* red) {
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(~0u, v, o);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    T s = 0;
    for (int i = 0; i < kThreads / 32; ++i) s += red[i];
    return s;
}
__device__ inline uint32_t block_xor(uint32_t v, uint32_t* red) {
    for (int o = 16; o; o >>= 1) v ^= __shfl_xor_sync(~0u, v, o);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    uint32_t s = 0;
    for (int i = 0; i < kThreads / 32; ++i) s ^= red[i];
    return s;
}
// exclusive prefix sum over the block in thread order; *total gets the sum
__device__ inline uint32_t block_exscan(uint32_t v, uint32_t* red, uint32_t* total) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    uint32_t x = v;
    for (int o = 1; o < 32; o <<= 1) {
        uint32_t y = __shfl_up_sync(~0u, x, o);
        if (lane >= o) x += y;
    }
    __syncthreads();
    if (lane == 31) red[wid] = x;
    __syncthreads();
    uint32_t before = 0, all = 0;
    for (int i = 0; i < kThreads / 32; ++i) {
        if (i < wid) before += red[i];
        all += red[i];
    }
    *total = all;
    return before + x - v;
}

// ---------------------------------------------------------------- deflate symbols
__device__ inline int len_code(int len) {            // 3..258 -> 0..28 (symbol 257 + code)
    int c = 0;
    while (c < 28 && c_len_base[c + 1] <= len) ++c;
    return len == 258 ? 28 : c;
}
__device__ inline int dist_code(int d) {             // 1..32768 -> 0..29
    if (d <= 4) return d - 1;
    const int l = 31 - __clz(d - 1);
    return 2 * l + (((d - 1) >> (l - 1)) & 1);
}
__device__ inline int dist_extra(int code) { return code < 4 ? 0 : (code >> 1) - 1; }
__device__ inline int dist_base(int code) { return code < 4 ? code + 1 : ((2 + (code & 1)) << ((code >> 1) - 1)) + 1; }
__device__ inline int fixed_lit_len(int s) { return s < 144 ? 8 : s < 256 ? 9 : s < 280 ? 7 : 8; }

__device__ inline void putbits(uint32_t* buf, uint32_t pos, uint32_t v, int n) {   // n <= 32, LSB first
    if (!n) return;
    const uint32_t w = pos >> 5, s = pos & 31;
    atomicOr(buf + w, v << s);
    if (s + n > 32) atomicOr(buf + w + 1, v >> (32 - s));
}

// ---------------------------------------------------------------- length-limited Huffman code lengths (one warp)
struct HuffScratch {
    uint32_t f[288];       // frequencies (unused symbols bumped so that at least two are coded)
    uint32_t nf[288];      // internal node weights
    int16_t sorted[288];   // used symbols by (frequency, symbol) ascending
    int16_t par[576];      // parent of leaf i (< m) / internal node m + k
    uint8_t depth[576];
    int bits[64];          // leaves per depth
};

// Code lengths for `nsym` symbols, none longer than `limit`: Huffman's two-queue construction over the symbols sorted by
// (frequency, symbol), then the depth histogram is brought under the limit (JPEG Annex K.3's adjustment) and the lengths
// are handed out again in frequency order.  Deterministic; called by all 32 lanes of one warp.
__device__ void huff_lengths(const uint32_t* freq, int nsym, int limit, uint8_t* len, HuffScratch& s) {
    const int lane = threadIdx.x & 31;
    for (int i = lane; i < nsym; i += 32) { s.f[i] = freq[i]; len[i] = 0; }
    for (int i = lane; i < 64; i += 32) s.bits[i] = 0;
    __syncwarp();
    if (lane == 0) {
        int used = 0;
        for (int i = 0; i < nsym; ++i) used += s.f[i] != 0;
        for (int i = 0; i < nsym && used < 2; ++i)
            if (!s.f[i]) { s.f[i] = 1; ++used; }
    }
    __syncwarp();
    for (int i = lane; i < nsym; i += 32) {
        const uint32_t fi = s.f[i];
        if (!fi) continue;
        int r = 0;
        for (int j = 0; j < nsym; ++j) {
            const uint32_t fj = s.f[j];
            r += fj && (fj < fi || (fj == fi && j < i));
        }
        s.sorted[r] = (int16_t)i;
    }
    __syncwarp();
    if (lane == 0) {
        int m = 0;
        for (int i = 0; i < nsym; ++i) m += s.f[i] != 0;
        int li = 0, ni = 0;
        for (int k = 0; k < m - 1; ++k) {
            uint32_t wsum = 0;
            for (int t = 0; t < 2; ++t) {
                const bool leaf = li < m && (ni >= k || s.f[s.sorted[li]] <= s.nf[ni]);
                const int node = leaf ? li++ : m + ni++;
                wsum += leaf ? s.f[s.sorted[node]] : s.nf[node - m];
                s.par[node] = (int16_t)(m + k);
            }
            s.nf[k] = wsum;
        }
        s.depth[2 * m - 2] = 0;
        for (int node = 2 * m - 3; node >= 0; --node) s.depth[node] = s.depth[s.par[node]] + 1;
        for (int i = 0; i < m; ++i) s.bits[min((int)s.depth[i], 63)]++;
        for (int i = 63; i > limit; --i)
            while (s.bits[i] > 0) {
                int j = i - 2;
                while (j > 0 && s.bits[j] == 0) --j;
                if (j == 0) break;
                s.bits[i] -= 2; s.bits[i - 1] += 1; s.bits[j + 1] += 2; s.bits[j] -= 1;
            }
        int k = 0;                                               // least frequent symbols get the longest codes
        for (int l = limit; l >= 1; --l)
            for (int c = 0; c < s.bits[l] && k < m; ++c) len[s.sorted[k++]] = (uint8_t)l;
    }
    __syncwarp();
}

// canonical codes (RFC 1951 3.2.2), bit-reversed for LSB-first emission; one thread
__device__ void canonical_codes(const uint8_t* len, int nsym, uint16_t* code, int* count, int* next) {
    for (int b = 0; b < 16; ++b) count[b] = 0;
    for (int i = 0; i < nsym; ++i) count[len[i]]++;
    count[0] = 0;
    int c = 0;
    for (int b = 1; b < 16; ++b) { c = (c + count[b - 1]) << 1; next[b] = c; }
    for (int i = 0; i < nsym; ++i)
        code[i] = len[i] ? (uint16_t)(__brev((uint32_t)next[len[i]]++) >> (32 - len[i])) : 0;
}

struct SegShared {
    uint32_t lhist[288], dhist[32], clhist[19];
    uint8_t llen[288], dlen[32], cllen[19];
    uint16_t lcode[288], dcode[32], clcode[19];
    uint16_t rle[320];          // code-length symbol | extra value << 5
    uint32_t crctab[256];
    unsigned long long red64[32];
    uint32_t red32[32];
    uint32_t x8[32];
    int count[16], next[16];
    int nrle, hlit, hdist, hclen, btype;   // btype: 0 stored, 1 fixed, 2 dynamic
    uint32_t header_bits;
};

__global__ void __launch_bounds__(kThreads, 1) k_deflate_segment(DeflateArgs a) {
    extern __shared__ __align__(16) uint8_t smem[];
    __shared__ SegShared sh;
    uint8_t* s_data = smem + kOffData;
    uint8_t* s_len = smem + kOffLen;
    uint16_t* s_dist = (uint16_t*)(smem + kOffDist);
    uint32_t* s_head = (uint32_t*)(smem + kOffHead);
    uint32_t* s_chosen = (uint32_t*)(smem + kOffChosen);
    uint32_t* s_out = (uint32_t*)(smem + kOffData);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int seg = blockIdx.x, img = blockIdx.y;
    const long long start = (long long)seg * kSeg;
    const int n = (int)min((long long)kSeg, a.len - start);
    const bool final_seg = seg == a.nseg - 1;
    const int avail = (int)min((long long)kWin, start);
    const int lo = kWin - avail;                               // first valid byte of s_data
    const uint8_t* src = a.scan + (size_t)img * a.len + start;

    for (int i = tid; i < avail + n; i += kThreads) s_data[lo + i] = src[i - avail];
    for (int i = tid; i < (1 << kHashBits); i += kThreads) s_head[i] = 0;
    for (int i = tid; i < kSeg / 32; i += kThreads) s_chosen[i] = 0;
    for (int i = tid; i < 288; i += kThreads) sh.lhist[i] = 0;
    if (tid < 32) sh.dhist[tid] = 0;
    if (tid < 19) sh.clhist[tid] = 0;
    if (tid < 32) sh.x8[tid] = a.x8[tid];
    crc_table(sh.crctab);
    __syncthreads();

    // ---- match search: hash heads hold the latest earlier position with the same 3-byte hash (atomicMax: order-free)
    const int end = kWin + n;
    auto hash3 = [&](int q) {
        const uint32_t v = s_data[q] | (uint32_t)s_data[q + 1] << 8 | (uint32_t)s_data[q + 2] << 16;
        return (v * 2654435761u) >> (32 - kHashBits);
    };
    for (int q = lo + tid; q < kWin && q + 2 < end; q += kThreads) atomicMax(s_head + hash3(q), (uint32_t)q + 1);
    __syncthreads();
    for (int r0 = 0; r0 < n; r0 += kThreads) {
        const int p = kWin + r0 + tid;
        const bool valid = r0 + tid < n, hashable = p + 2 < end;
        const uint32_t hsh = hashable ? hash3(p) : 0;
        const uint32_t cand = hashable ? s_head[hsh] : 0;      // a position before this round
        __syncthreads();
        if (hashable) atomicMax(s_head + hsh, (uint32_t)p + 1);
        if (valid) {
            const int maxlen = min(258, end - p);
            int best = 0, bestd = 0;
#pragma unroll
            for (int ci = 0; ci < 4; ++ci) {       // left byte, left pixel, row above, hash head
                const int d = ci == 0 ? 1 : ci == 1 ? a.bpp : ci == 2 ? a.stride : cand ? p - (int)(cand - 1) : 0;
                if (best == maxlen || d < 1 || d > kWin || p - d < lo || (ci == 1 && d == 1)) continue;
                const uint8_t* x = s_data + p;
                const uint8_t* y = x - d;
                int l = 0;
                while (l < maxlen && x[l] == y[l]) ++l;
                if (l > best) { best = l; bestd = d; }
            }
            s_len[r0 + tid] = (uint8_t)(best >= 3 ? best - 3 : 0);
            s_dist[r0 + tid] = (uint16_t)(best >= 3 ? bestd : 0);
        }
        __syncthreads();
    }

    // ---- greedy parse, left to right, by one warp: a ballot skips runs of literals 32 positions at a time
    if (warp == 0) {
        int p = 0;
        while (p < n) {
            const int q = p + lane;
            const unsigned m = __ballot_sync(~0u, q < n && s_dist[q] != 0);
            const int k = m ? __ffs(m) - 1 : 32;
            if (q < n && lane <= k) atomicOr(s_chosen + (q >> 5), 1u << (q & 31));
            p = m ? p + k + 3 + s_len[p + k] : p + 32;
        }
    }
    __syncthreads();

    // ---- histograms of the chosen tokens (integer counts: order-free)
    const int p0 = tid * kPer;
    for (int q = p0; q < min(p0 + kPer, n); ++q) {
        if (!((s_chosen[q >> 5] >> (q & 31)) & 1)) continue;
        if (s_dist[q]) {
            atomicAdd(sh.lhist + 257 + len_code(s_len[q] + 3), 1u);
            atomicAdd(sh.dhist + dist_code(s_dist[q]), 1u);
        } else {
            atomicAdd(sh.lhist + s_data[kWin + q], 1u);
        }
    }
    if (tid == 0) atomicAdd(sh.lhist + 256, 1u);               // end of block
    __syncthreads();

    // ---- codes: literal/length on warp 0, distance on warp 1 (scratch in the dead hash table), then the header
    HuffScratch* hs = (HuffScratch*)s_head;
    if (warp == 0) huff_lengths(sh.lhist, 286, 15, sh.llen, hs[0]);
    if (warp == 1) huff_lengths(sh.dhist, 30, 15, sh.dlen, hs[1]);
    __syncthreads();
    if (warp == 0) {
        if (lane == 0) {
            int hlit = 286, hdist = 30;
            while (hlit > 257 && !sh.llen[hlit - 1]) --hlit;
            while (hdist > 1 && !sh.dlen[hdist - 1]) --hdist;
            const int total = hlit + hdist;
            auto L = [&](int i) { return i < hlit ? sh.llen[i] : sh.dlen[i - hlit]; };
            int nr = 0;
            auto emit = [&](int sym, int extra) { sh.rle[nr++] = (uint16_t)(sym | extra << 5); sh.clhist[sym]++; };
            for (int i = 0; i < total;) {
                const int v = L(i);
                int run = 1;
                while (i + run < total && L(i + run) == v) ++run;
                i += run;
                if (v == 0) {
                    for (; run >= 11; ) { const int r = min(run, 138); emit(18, r - 11); run -= r; }
                    if (run >= 3) { emit(17, run - 3); run = 0; }
                } else {
                    emit(v, 0); --run;
                    for (; run >= 3; ) { const int r = min(run, 6); emit(16, r - 3); run -= r; }
                }
                for (; run > 0; --run) emit(v, 0);
            }
            sh.nrle = nr; sh.hlit = hlit; sh.hdist = hdist;
        }
        __syncwarp();
        huff_lengths(sh.clhist, 19, 7, sh.cllen, hs[0]);
        if (lane == 0) {
            int hclen = 19;
            while (hclen > 4 && !sh.cllen[c_cl_order[hclen - 1]]) --hclen;
            sh.hclen = hclen;
            unsigned long long hdr = 3 + 5 + 5 + 4 + 3 * hclen, dyn = 0, fix = 3, extra = 0;
            for (int i = 0; i < sh.nrle; ++i) {
                const int sym = sh.rle[i] & 31;
                hdr += sh.cllen[sym] + (sym == 16 ? 2 : sym == 17 ? 3 : sym == 18 ? 7 : 0);
            }
            for (int i = 0; i < 286; ++i) {
                dyn += (unsigned long long)sh.lhist[i] * sh.llen[i];
                fix += (unsigned long long)sh.lhist[i] * fixed_lit_len(i);
                if (i >= 257) extra += (unsigned long long)sh.lhist[i] * c_len_extra[i - 257];
            }
            for (int i = 0; i < 30; ++i) {
                dyn += (unsigned long long)sh.dhist[i] * sh.dlen[i];
                fix += (unsigned long long)sh.dhist[i] * 5;
                extra += (unsigned long long)sh.dhist[i] * dist_extra(i);
            }
            dyn += hdr + extra;
            fix += extra;
            const int flush = final_seg ? 0 : 3;             // the sync flush's block header shares the last byte
            const unsigned long long by_dyn = (dyn + flush + 7) / 8, by_fix = (fix + flush + 7) / 8, by_sto = 5 + (unsigned long long)n;
            int bt = 2;
            if (by_fix <= by_dyn) bt = 1;
            if (by_sto < (bt == 2 ? by_dyn : by_fix)) bt = 0;
            if (bt == 1) {
                for (int i = 0; i < 288; ++i) sh.llen[i] = (uint8_t)fixed_lit_len(i);
                for (int i = 0; i < 30; ++i) sh.dlen[i] = 5;
            }
            sh.btype = bt;
            sh.header_bits = bt == 2 ? (uint32_t)hdr : 3;
            canonical_codes(sh.llen, bt == 1 ? 288 : 286, sh.lcode, sh.count, sh.next);   // fixed: 286, 287 precede the 9-bit codes
            canonical_codes(sh.dlen, 30, sh.dcode, sh.count, sh.next);
            canonical_codes(sh.cllen, 19, sh.clcode, sh.count, sh.next);
        }
    }
    __syncthreads();

    // ---- emission: per-token bit offsets from a block scan; each thread ORs its tokens into the zeroed buffer
    const int bt = sh.btype;
    for (int i = tid; i < kOutWords; i += kThreads) s_out[i] = 0;    // the window bytes are dead from here on
    uint32_t mybits = 0;
    if (bt != 0)
        for (int q = p0; q < min(p0 + kPer, n); ++q) {
            if (!((s_chosen[q >> 5] >> (q & 31)) & 1)) continue;
            if (s_dist[q]) {
                const int lc = len_code(s_len[q] + 3), dc = dist_code(s_dist[q]);
                mybits += sh.llen[257 + lc] + c_len_extra[lc] + sh.dlen[dc] + dist_extra(dc);
            } else {
                mybits += sh.llen[s_data[kWin + q]];
            }
        }
    uint32_t tok_bits;
    uint32_t pos = sh.header_bits + block_exscan(mybits, sh.red32, &tok_bits);   // block_exscan syncs: the zeroing is done
    uint8_t* ob = (uint8_t*)s_out;
    uint32_t nbytes;
    if (bt == 0) {
        nbytes = 5 + n + (final_seg ? 0 : 5);
        for (int i = tid; i < n; i += kThreads) ob[5 + i] = s_data[kWin + i];
        if (tid == 0) {
            ob[0] = final_seg ? 1 : 0;
            ob[1] = n & 255; ob[2] = n >> 8; ob[3] = ~n & 255; ob[4] = (~n >> 8) & 255;
            if (!final_seg) { ob[5 + n] = 0; ob[6 + n] = 0; ob[7 + n] = 0; ob[8 + n] = 0xff; ob[9 + n] = 0xff; }
        }
    } else {
        for (int q = p0; q < min(p0 + kPer, n); ++q) {
            if (!((s_chosen[q >> 5] >> (q & 31)) & 1)) continue;
            if (s_dist[q]) {
                const int len = s_len[q] + 3, d = s_dist[q];
                const int lc = len_code(len), dc = dist_code(d);
                const int ll = sh.llen[257 + lc], le = c_len_extra[lc], dl = sh.dlen[dc], de = dist_extra(dc);
                putbits(s_out, pos, sh.lcode[257 + lc] | (uint32_t)(len - c_len_base[lc]) << ll, ll + le);
                putbits(s_out, pos + ll + le, sh.dcode[dc] | (uint32_t)(d - dist_base(dc)) << dl, dl + de);
                pos += ll + le + dl + de;
            } else {
                const int s = s_data[kWin + q];
                putbits(s_out, pos, sh.lcode[s], sh.llen[s]);
                pos += sh.llen[s];
            }
        }
        const uint32_t eob = sh.header_bits + tok_bits;
        if (tid == 0) {
            putbits(s_out, 0, (final_seg ? 1u : 0u) | (uint32_t)bt << 1, 3);
            if (bt == 2) {
                uint32_t hp = 3;
                putbits(s_out, hp, sh.hlit - 257, 5); hp += 5;
                putbits(s_out, hp, sh.hdist - 1, 5); hp += 5;
                putbits(s_out, hp, sh.hclen - 4, 4); hp += 4;
                for (int i = 0; i < sh.hclen; ++i, hp += 3) putbits(s_out, hp, sh.cllen[c_cl_order[i]], 3);
                for (int i = 0; i < sh.nrle; ++i) {
                    const int sym = sh.rle[i] & 31, ex = sh.rle[i] >> 5, eb = sym == 16 ? 2 : sym == 17 ? 3 : sym == 18 ? 7 : 0;
                    putbits(s_out, hp, sh.clcode[sym] | (uint32_t)ex << sh.cllen[sym], sh.cllen[sym] + eb);
                    hp += sh.cllen[sym] + eb;
                }
            }
            putbits(s_out, eob, sh.lcode[256], sh.llen[256]);
        }
        const uint32_t bits = eob + sh.llen[256];
        nbytes = final_seg ? (bits + 7) / 8 : (bits + 3 + 7) / 8 + 4;
        __syncthreads();
        if (tid == 0 && !final_seg) { ob[nbytes - 2] = 0xff; ob[nbytes - 1] = 0xff; }   // sync flush: empty stored block
    }
    __syncthreads();

    // ---- out: the segment's bytes, their raw CRC (init 0, combined over thread chunks) and the Adler-32 partials
    const size_t slot = (size_t)img * a.nseg + seg;
    uint32_t* dst = (uint32_t*)(a.slots + slot * kSlot);
    for (int i = tid; i < (int)(nbytes + 3) / 4; i += kThreads) dst[i] = s_out[i];
    const int cs = (nbytes + kThreads - 1) / kThreads;
    const int c0 = min((int)nbytes, tid * cs), c1 = min((int)nbytes, c0 + cs);
    const uint32_t part = gf2_mul(x8pow(sh.x8, nbytes - c1), crc_bytes(sh.crctab, 0, ob + c0, c1 - c0));
    const uint32_t crc = block_xor(part, sh.red32);
    unsigned long long s1 = 0, s2 = 0;
    for (int q = p0; q < min(p0 + kPer, n); ++q) {
        const uint32_t b = s_data[kWin + q];
        s1 += b;
        s2 += (unsigned long long)(n - q) * b;
    }
    s1 = block_sum(s1, sh.red64);
    s2 = block_sum(s2, sh.red64);
    if (tid == 0) {
        uint32_t* m = a.meta + slot * 4;
        m[0] = nbytes; m[1] = crc; m[2] = (uint32_t)(s1 % kAdlerMod); m[3] = (uint32_t)(s2 % kAdlerMod);
    }
}

__device__ inline void put_be32(uint8_t* p, uint32_t v) { p[0] = v >> 24; p[1] = v >> 16; p[2] = v >> 8; p[3] = v; }

__global__ void __launch_bounds__(kThreads, 1) k_png_assemble(AssembleArgs a) {
    __shared__ uint32_t s_tab[256], s_off[kThreads], s_len[kThreads], red32[32], s_x8[32];
    __shared__ unsigned long long red64[32];
    const int tid = threadIdx.x, img = blockIdx.x;
    const uint32_t* meta = a.meta + (size_t)img * a.nseg * 4;
    const uint8_t* slots = a.slots + (size_t)img * a.nseg * kSlot;
    uint8_t* out = a.out + (size_t)img * a.out_stride;
    crc_table(s_tab);
    if (tid < 32) s_x8[tid] = a.x8[tid];
    unsigned long long t = 0;
    for (int k = tid; k < a.nseg; k += kThreads) t += meta[4 * k];
    const unsigned long long total = block_sum(t, red64);       // deflate bytes

    // stream CRC of the segments: sum over k of crc_k * x^(8 * bytes after k); Adler-32: sum over k of the partials with
    // the weighted sum shifted by the input bytes after k
    uint32_t cx = 0;
    unsigned long long A = 0, B = 0, carry = 0;
    for (int base = 0; base < a.nseg; base += kThreads) {
        const int k = base + tid;
        const uint32_t bytes = k < a.nseg ? meta[4 * k] : 0;
        uint32_t chunk;
        const uint32_t off = block_exscan(bytes, red32, &chunk);
        if (k < a.nseg) {
            const unsigned long long o = carry + off;
            s_off[tid] = (uint32_t)o; s_len[tid] = bytes;
            cx ^= gf2_mul(x8pow(s_x8, total - o - bytes), meta[4 * k + 1]);
            const long long in0 = (long long)k * kSeg, in_n = min((long long)kSeg, a.len - in0);
            const unsigned long long S = meta[4 * k + 2], T = meta[4 * k + 3];
            A = (A + S) % kAdlerMod;
            B = (B + T + S * (unsigned long long)((a.len - in0 - in_n) % kAdlerMod)) % kAdlerMod;
        }
        carry += chunk;
        __syncthreads();
        const int nk = min(kThreads, a.nseg - base);
        for (int j = 0; j < nk; ++j) {
            const uint8_t* s = slots + (size_t)(base + j) * kSlot;
            uint8_t* d = out + kHeadBytes + s_off[j];
            for (int i = tid; i < (int)s_len[j]; i += kThreads) d[i] = s[i];
        }
        __syncthreads();
    }
    cx = block_xor(cx, red32);
    A = block_sum(A, red64) % kAdlerMod;
    B = block_sum(B, red64) % kAdlerMod;
    if (tid == 0) {
        const uint32_t adler = (uint32_t)(((B + (unsigned long long)(a.len % kAdlerMod)) % kAdlerMod) << 16 | ((1 + A) % kAdlerMod));
        put_be32(out, 0x89504e47u); put_be32(out + 4, 0x0d0a1a0au);                    // signature
        uint8_t* ih = out + 8;
        put_be32(ih, 13);
        ih[4] = 'I'; ih[5] = 'H'; ih[6] = 'D'; ih[7] = 'R';
        put_be32(ih + 8, (uint32_t)a.w); put_be32(ih + 12, (uint32_t)a.h);
        ih[16] = 8; ih[17] = a.c == 1 ? 0 : a.c == 3 ? 2 : 6; ih[18] = ih[19] = ih[20] = 0;
        put_be32(ih + 21, ~crc_bytes(s_tab, ~0u, ih + 4, 17));
        uint8_t* id = out + 33;
        put_be32(id, (uint32_t)(2 + total + 4));
        id[4] = 'I'; id[5] = 'D'; id[6] = 'A'; id[7] = 'T'; id[8] = 0x78; id[9] = 0x01;   // CMF/FLG: deflate, 32 KB window
        uint32_t crc = gf2_mul(x8pow(s_x8, total), crc_bytes(s_tab, ~0u, id + 4, 6)) ^ cx;
        uint8_t* tl = out + kHeadBytes + total;
        put_be32(tl, adler);
        crc = ~crc_bytes(s_tab, crc, tl, 4);
        put_be32(tl + 4, crc);
        put_be32(tl + 8, 0); put_be32(tl + 12, 0x49454e44u); put_be32(tl + 16, 0xae426082u);   // IEND
        a.out_lens[img] = kHeadBytes + total + kTailBytes;
    }
}

// the stream bytes of one image inside the envelope, else 0 (each factor bounded before it is multiplied)
size_t stream_bytes(int h, int w, int c) {
    if (h < 1 || w < 1 || !(c == 1 || c == 3 || c == 4)) return 0;
    if ((size_t)w > (kMaxStream - 1) / (size_t)c) return 0;
    const size_t row = 1 + (size_t)w * c;
    if ((size_t)h > kMaxStream / row) return 0;
    return (size_t)h * row;
}
size_t n_segments(size_t len) { return (len + kSeg - 1) / kSeg; }

void x8_table(uint32_t* x8) {
    uint32_t p = 0x80000000u >> 8;                               // x^8
    for (int k = 0; k < 32; ++k) { x8[k] = p; p = gf2_mul(p, p); }
}

}  // namespace
}  // namespace p3d

using namespace p3d;

extern "C" size_t p3d_png_device_bound(int32_t h, int32_t w, int32_t channels) {
    const size_t len = stream_bytes(h, w, channels);
    return len ? kHeadBytes + kTailBytes + len + 10 * n_segments(len) : 0;
}

extern "C" size_t p3d_png_device_workspace_bytes(int32_t n, int32_t h, int32_t w, int32_t channels) {
    const size_t len = stream_bytes(h, w, channels);
    if (!len || n < 1 || n > kMaxImages) return 0;
    return (size_t)n * n_segments(len) * (kSlot + 16);
}

extern "C" int p3d_png_encode_device(const uint8_t* scanlines, int32_t n, int32_t h, int32_t w, int32_t channels,
                                     void* workspace, size_t workspace_bytes, uint8_t* out, size_t out_stride,
                                     uint64_t* out_lens, void* stream) {
    P3D_REQUIRE(scanlines && workspace && out && out_lens, "p3d_png_encode_device: NULL pointer");
    const size_t len = stream_bytes(h, w, channels);
    P3D_REQUIRE(len && n >= 1 && n <= kMaxImages,
                "p3d_png_encode_device: n=%d h=%d w=%d c=%d outside the envelope (n <= %d, C in {1,3,4}, h*(1+w*C) <= %zu)",
                n, h, w, channels, kMaxImages, kMaxStream);
    const size_t need = p3d_png_device_workspace_bytes(n, h, w, channels), bound = p3d_png_device_bound(h, w, channels);
    if (workspace_bytes < need) {
        set_error("p3d_png_encode_device: workspace of %zu bytes, %zu needed", workspace_bytes, need);
        return P3D_EWORKSPACE;
    }
    P3D_REQUIRE(out_stride >= bound && out_stride <= SIZE_MAX / (size_t)n,
                "p3d_png_encode_device: out_stride %zu (at least the bound %zu, and n * stride must not wrap)", out_stride, bound);
    const int nseg = (int)n_segments(len);
    DeflateArgs d;
    d.scan = scanlines; d.slots = (uint8_t*)workspace; d.meta = (uint32_t*)((uint8_t*)workspace + (size_t)n * nseg * kSlot);
    d.len = (long long)len; d.nseg = nseg; d.bpp = channels; d.stride = (int)(len / h);
    static uint32_t x8[32];
    static bool x8_ready = [] { x8_table(x8); return true; }();
    (void)x8_ready;
    memcpy(d.x8, x8, sizeof(x8));
    cudaStream_t st = (cudaStream_t)stream;
    P3D_CUDA_TRY(cudaFuncSetAttribute(k_deflate_segment, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem));
    k_deflate_segment<<<dim3((unsigned)nseg, (unsigned)n), kThreads, kSmem, st>>>(d);
    P3D_LAUNCH_CHECK();
    AssembleArgs as;
    as.slots = d.slots; as.meta = d.meta; as.out = out; as.out_stride = out_stride; as.out_lens = (uint64_t*)out_lens;
    as.len = d.len; as.nseg = nseg; as.h = h; as.w = w; as.c = channels;
    memcpy(as.x8, x8, sizeof(x8));
    k_png_assemble<<<(unsigned)n, kThreads, 0, st>>>(as);
    P3D_LAUNCH_CHECK();
    return P3D_OK;
}
