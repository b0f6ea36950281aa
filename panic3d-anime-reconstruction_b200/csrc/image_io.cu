// Image output path (SURVEY 8f-4): device-side quantisation + PNG scan-line filtering, host-side deflate / file writing on
// a thread pool.  Replaces the blocking `I(tensor).save(fn)` at the end of every view of the reference's eval sweep
// (_scripts/eval/generate.py:141-148 -> _util/twodee_v1.py:174-185 `to_pil_image(clamp(0,1))` -> PIL PNG encoder).
//
// Byte work, HBM/PCIe-bound: no tensor cores.  One warp per scan-line: the raw row and the row above are quantised into
// shared memory once, the five PNG filters are scored with libpng's minimum-sum-of-absolute-differences heuristic by a warp
// reduction, and the chosen filter's bytes are written behind the filter-type byte.  What crosses PCIe is the filtered
// 8-bit stream (4x less than the fp32 image); zlib's deflate (inherently serial per stream) runs on host threads.
#include <zlib.h>

#include <algorithm>
#include <condition_variable>
#include <deque>
#include <mutex>
#include <thread>
#include <vector>

#include "p3d_common.cuh"
#include "../../include/p3d_imageio.h"

namespace p3d {
namespace {

struct QuantArgs {
    const float *image, *extra;
    int n, c, c_img, h, w;
    float scale[4], shift[4];
    int affine;
};

__device__ __forceinline__ unsigned int quant_u8(const QuantArgs& a, int n, int ch, int y, int x) {
    float v = ch < a.c_img ? __ldg(a.image + (((size_t)n * a.c_img + ch) * a.h + y) * a.w + x)
                           : __ldg(a.extra + ((size_t)n * a.h + y) * a.w + x);
    if (a.affine) v = (v + a.shift[ch]) * a.scale[ch];
    v = fminf(fmaxf(v, 0.f), 1.f);                       // clamp(0,1); NaN -> 0
    return (unsigned int)(int)(v * 255.f);               // .mul(255).byte(): truncation
}

__device__ __forceinline__ int paeth(int a, int b, int c) {
    int p = a + b - c, pa = abs(p - a), pb = abs(p - b), pc = abs(p - c);
    return (pa <= pb && pa <= pc) ? a : (pb <= pc ? b : c);
}
__device__ __forceinline__ int filt(int type, int x, int a, int b, int c) {
    int r = type == 0 ? x : type == 1 ? x - a : type == 2 ? x - b : type == 3 ? x - ((a + b) >> 1) : x - paeth(a, b, c);
    return r & 255;
}

// one warp per scan-line; dynamic smem: warps_per_block * 2 * rowbytes
__global__ void k_png_scanlines(QuantArgs a, unsigned char* __restrict__ out, int warps_per_block) {
    extern __shared__ unsigned char s_rows[];
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    const long long row = (long long)blockIdx.x * warps_per_block + wib;
    if (row >= (long long)a.n * a.h) return;
    const int n = (int)(row / a.h), y = (int)(row - (long long)n * a.h);
    const int rb = a.w * a.c, bpp = a.c;
    unsigned char* cur = s_rows + (size_t)wib * 2 * rb;
    unsigned char* prev = cur + rb;
    for (int ch = 0; ch < a.c; ++ch)
        for (int x = lane; x < a.w; x += 32) {
            cur[x * a.c + ch] = (unsigned char)quant_u8(a, n, ch, y, x);
            prev[x * a.c + ch] = y > 0 ? (unsigned char)quant_u8(a, n, ch, y - 1, x) : (unsigned char)0;
        }
    __syncwarp();
    // score the five filters: sum over the row of |filtered byte as int8| (libpng png_write_find_filter)
    unsigned int s0 = 0, s1 = 0, s2 = 0, s3 = 0, s4 = 0;
    for (int i = lane; i < rb; i += 32) {
        int x = cur[i], b = prev[i], l = i >= bpp ? cur[i - bpp] : 0, ul = i >= bpp ? prev[i - bpp] : 0;
        int f;
        f = filt(0, x, l, b, ul); s0 += f < 128 ? f : 256 - f;
        f = filt(1, x, l, b, ul); s1 += f < 128 ? f : 256 - f;
        f = filt(2, x, l, b, ul); s2 += f < 128 ? f : 256 - f;
        f = filt(3, x, l, b, ul); s3 += f < 128 ? f : 256 - f;
        f = filt(4, x, l, b, ul); s4 += f < 128 ? f : 256 - f;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        s0 += __shfl_xor_sync(0xffffffffu, s0, o); s1 += __shfl_xor_sync(0xffffffffu, s1, o); s2 += __shfl_xor_sync(0xffffffffu, s2, o);
        s3 += __shfl_xor_sync(0xffffffffu, s3, o); s4 += __shfl_xor_sync(0xffffffffu, s4, o);
    }
    int type = 0; unsigned int best = s0;                 // first minimum in the order none, sub, up, average, paeth
    if (s1 < best) { best = s1; type = 1; }
    if (s2 < best) { best = s2; type = 2; }
    if (s3 < best) { best = s3; type = 3; }
    if (s4 < best) { best = s4; type = 4; }
    unsigned char* dst = out + (size_t)row * (1 + rb);
    if (lane == 0) dst[0] = (unsigned char)type;
    for (int i = lane; i < rb; i += 32) {
        int x = cur[i], b = prev[i], l = i >= bpp ? cur[i - bpp] : 0, ul = i >= bpp ? prev[i - bpp] : 0;
        dst[1 + i] = (unsigned char)filt(type, x, l, b, ul);
    }
}

// rows too long for the shared-memory staging: filter type 0 (none); also the plain NHWC u8 output (prefix == 0)
__global__ void k_quantize_nhwc(QuantArgs a, unsigned char* __restrict__ out, int prefix) {
    const long long total = (long long)a.n * a.h * a.w;
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int x = (int)(i % a.w);
    const long long r = i / a.w;
    const int y = (int)(r % a.h), n = (int)(r / a.h);
    unsigned char* dst = out + (size_t)r * (prefix + a.w * a.c) + prefix + (size_t)x * a.c;
    if (prefix && x == 0) dst[-1] = 0;
    for (int ch = 0; ch < a.c; ++ch) dst[ch] = (unsigned char)quant_u8(a, n, ch, y, x);
}

int fill_args(QuantArgs& a, const float* image, const float* extra, int n, int c, int h, int w, const float* scale, const float* shift) {
    P3D_REQUIRE(image != nullptr, "p3d_image: image is NULL");
    P3D_REQUIRE(c == 1 || c == 3 || c == 4, "p3d_image: %d channels (PNG modes L / RGB / RGBA need 1, 3 or 4)", c);
    P3D_REQUIRE(n > 0 && h > 0 && w > 0, "p3d_image: bad shape n=%d h=%d w=%d", n, h, w);
    P3D_REQUIRE(!(extra && c == 1), "p3d_image: an extra plane needs at least one image plane in front of it");
    P3D_REQUIRE((scale == nullptr) == (shift == nullptr), "p3d_image: scale and shift come together");
    a.image = image; a.extra = extra; a.n = n; a.c = c; a.c_img = extra ? c - 1 : c; a.h = h; a.w = w;
    a.affine = scale != nullptr;
    for (int i = 0; i < 4; ++i) { a.scale[i] = scale && i < c ? scale[i] : 1.f; a.shift[i] = shift && i < c ? shift[i] : 0.f; }
    return P3D_OK;
}

// ---------------------------------------------------------------- host: PNG container
void put_be32(unsigned char* p, uint32_t v) { p[0] = v >> 24; p[1] = v >> 16; p[2] = v >> 8; p[3] = v; }
size_t put_chunk(unsigned char* p, const char* type, const unsigned char* data, size_t len) {
    put_be32(p, (uint32_t)len);
    memcpy(p + 4, type, 4);
    if (len && data != p + 8) memcpy(p + 8, data, len);
    uLong crc = crc32(0L, Z_NULL, 0);
    crc = crc32(crc, p + 4, (uInt)(4 + len));
    put_be32(p + 8 + len, (uint32_t)crc);
    return 12 + len;
}
size_t encode_bound(int h, int w, int c) { return 8 + 25 + 12 + compressBound((uLong)h * (1 + (uLong)w * c)) + 12; }

int encode(const unsigned char* scan, int h, int w, int c, int level, unsigned char* out, size_t cap, size_t* out_len) {
    const size_t need = encode_bound(h, w, c);
    if (out_len) *out_len = need;
    if (cap < need) { set_error("p3d_png_encode: output buffer of %zu bytes, %zu needed", cap, need); return P3D_EWORKSPACE; }
    static const unsigned char sig[8] = {0x89, 'P', 'N', 'G', 0x0d, 0x0a, 0x1a, 0x0a};
    memcpy(out, sig, 8);
    size_t o = 8;
    unsigned char ihdr[13];
    put_be32(ihdr, (uint32_t)w); put_be32(ihdr + 4, (uint32_t)h);
    ihdr[8] = 8; ihdr[9] = c == 1 ? 0 : c == 3 ? 2 : 6; ihdr[10] = ihdr[11] = ihdr[12] = 0;
    o += put_chunk(out + o, "IHDR", ihdr, 13);
    uLongf zlen = (uLongf)(cap - o - 12 - 12);
    int rc = compress2(out + o + 8, &zlen, scan, (uLong)h * (1 + (uLong)w * c), level);
    if (rc != Z_OK) { set_error("p3d_png_encode: zlib compress2 failed (%d)", rc); return P3D_EINVAL; }
    o += put_chunk(out + o, "IDAT", out + o + 8, zlen);
    o += put_chunk(out + o, "IEND", nullptr, 0);
    if (out_len) *out_len = o;
    return P3D_OK;
}

// ---------------------------------------------------------------- host: asynchronous writer
struct Job {
    std::string path;
    int h, w, c;
    unsigned char* host;          // staging (pinned when `pinned`)
    size_t bytes, cap;
    bool pinned;
    cudaEvent_t ev = nullptr;     // D2H copy done (nullptr for host submissions)
    int device;
    bool encoded = false;         // host holds [u64 length | file bytes] from p3d_png_encode_device
};

struct Writer {
    std::vector<std::thread> threads;
    std::mutex m;
    std::condition_variable cv_work, cv_done;
    std::deque<Job> q;
    std::vector<std::pair<unsigned char*, size_t>> pinned_free;     // staging buffers ready for reuse
    int inflight = 0, failed = 0, level = 3;
    bool stop = false;
    std::string first_error;

    void fail(const std::string& msg) {
        std::lock_guard<std::mutex> lk(m);
        if (failed++ == 0) first_error = msg;
    }
    void run() {
        std::vector<unsigned char> png;
        for (;;) {
            Job j;
            {
                std::unique_lock<std::mutex> lk(m);
                cv_work.wait(lk, [&] { return stop || !q.empty(); });
                if (q.empty()) return;
                j = std::move(q.front());
                q.pop_front();
            }
            bool ok = true;
            if (j.ev) {
                cudaSetDevice(j.device);
                cudaError_t e = cudaEventSynchronize(j.ev);
                cudaEventDestroy(j.ev);
                if (e != cudaSuccess) { fail(std::string("copy of ") + j.path + " failed: " + cudaGetErrorString(e)); ok = false; }
            }
            if (ok) {
                const unsigned char* file = png.data();
                size_t len = 0;
                if (j.encoded) {
                    memcpy(&len, j.host, sizeof(uint64_t));
                    file = j.host + sizeof(uint64_t);
                    if (len > j.bytes - sizeof(uint64_t)) { fail("encoded " + j.path + " is longer than its bound"); ok = false; }
                } else {
                    png.resize(encode_bound(j.h, j.w, j.c));
                    if (encode(j.host, j.h, j.w, j.c, level, png.data(), png.size(), &len) != P3D_OK) { fail("encoding " + j.path + " failed"); ok = false; }
                    file = png.data();
                }
                if (ok) {
                    const std::string tmp = j.path + ".tmp";
                    FILE* f = fopen(tmp.c_str(), "wb");
                    if (!f || fwrite(file, 1, len, f) != len || fclose(f) != 0 || rename(tmp.c_str(), j.path.c_str()) != 0) {
                        if (f) remove(tmp.c_str());
                        fail("cannot write " + j.path);
                    }
                }
            }
            {
                std::lock_guard<std::mutex> lk(m);
                if (j.pinned) pinned_free.emplace_back(j.host, j.cap); else free(j.host);
                --inflight;
            }
            cv_done.notify_all();
        }
    }
};

int check_image(const void* w, const void* src, int h, int wd, int c, const char* path) {
    P3D_REQUIRE(w && src && path && path[0], "p3d_png_writer_submit: NULL writer, source or path");
    P3D_REQUIRE(h > 0 && wd > 0 && (c == 1 || c == 3 || c == 4), "p3d_png_writer_submit: bad image h=%d w=%d c=%d", h, wd, c);
    return P3D_OK;
}

}  // namespace
}  // namespace p3d

using namespace p3d;

extern "C" size_t p3d_png_scanline_bytes(int32_t h, int32_t w, int32_t channels) {
    return (h > 0 && w > 0 && channels > 0) ? (size_t)h * (1 + (size_t)w * channels) : 0;
}

extern "C" int p3d_image_to_png_scanlines(const float* image, const float* extra, int32_t n, int32_t c, int32_t h, int32_t w,
                                          const float* scale, const float* shift, uint8_t* scanlines, void* stream) {
    QuantArgs a;
    if (int rc = fill_args(a, image, extra, n, c, h, w, scale, shift)) return rc;
    P3D_REQUIRE(scanlines != nullptr, "p3d_image_to_png_scanlines: output is NULL");
    const size_t rb = (size_t)w * c;
    int wpb = (int)std::min<size_t>(8, (200 * 1024) / (2 * rb));
    if (wpb < 1) {                                               // rows beyond the shared-memory staging: filter 0
        const long long total = (long long)n * h * w;
        k_quantize_nhwc<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(a, scanlines, 1);
        P3D_LAUNCH_CHECK();
        return P3D_OK;
    }
    const size_t smem = (size_t)wpb * 2 * rb;
    if (smem > 48 * 1024) P3D_CUDA_TRY(cudaFuncSetAttribute(k_png_scanlines, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const long long rows = (long long)n * h;
    k_png_scanlines<<<(unsigned)((rows + wpb - 1) / wpb), wpb * 32, smem, (cudaStream_t)stream>>>(a, scanlines, wpb);
    P3D_LAUNCH_CHECK();
    return P3D_OK;
}

extern "C" int p3d_image_to_u8(const float* image, const float* extra, int32_t n, int32_t c, int32_t h, int32_t w,
                               const float* scale, const float* shift, uint8_t* out_nhwc, void* stream) {
    QuantArgs a;
    if (int rc = fill_args(a, image, extra, n, c, h, w, scale, shift)) return rc;
    P3D_REQUIRE(out_nhwc != nullptr, "p3d_image_to_u8: output is NULL");
    const long long total = (long long)n * h * w;
    k_quantize_nhwc<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(a, out_nhwc, 0);
    P3D_LAUNCH_CHECK();
    return P3D_OK;
}

extern "C" size_t p3d_png_encode_bound(int32_t h, int32_t w, int32_t channels) {
    return (h > 0 && w > 0 && channels > 0) ? encode_bound(h, w, channels) : 0;
}

extern "C" int p3d_png_encode_host(const uint8_t* scanlines, int32_t h, int32_t w, int32_t channels, int32_t level,
                                   uint8_t* out, size_t cap, size_t* out_len) {
    P3D_REQUIRE(scanlines && out, "p3d_png_encode_host: NULL pointer");
    P3D_REQUIRE(h > 0 && w > 0 && (channels == 1 || channels == 3 || channels == 4), "p3d_png_encode_host: bad image h=%d w=%d c=%d", h, w, channels);
    P3D_REQUIRE(level >= 0 && level <= 9, "p3d_png_encode_host: zlib level %d outside 0..9", level);
    return encode(scanlines, h, w, channels, level, out, cap, out_len);
}

extern "C" int p3d_png_writer_create(int32_t n_threads, int32_t compress_level, void** writer) {
    P3D_REQUIRE(writer != nullptr, "p3d_png_writer_create: NULL handle pointer");
    P3D_REQUIRE(n_threads >= 1 && n_threads <= 256, "p3d_png_writer_create: %d threads", n_threads);
    P3D_REQUIRE(compress_level >= 0 && compress_level <= 9, "p3d_png_writer_create: zlib level %d outside 0..9", compress_level);
    Writer* w = new Writer();
    w->level = compress_level;
    for (int i = 0; i < n_threads; ++i) w->threads.emplace_back([w] { w->run(); });
    *writer = w;
    return P3D_OK;
}

namespace p3d {
namespace {

// D2H copies of `n` (pointer, bytes) pieces, back to back into the writer's pinned staging, then the job is queued
int submit_device(Writer* wr, Job& j, const void* const* src, const size_t* bytes, int n, cudaStream_t stream) {
    j.bytes = 0;
    for (int i = 0; i < n; ++i) j.bytes += bytes[i];
    j.pinned = true; j.host = nullptr; j.cap = 0;
    {
        std::lock_guard<std::mutex> lk(wr->m);
        for (size_t i = 0; i < wr->pinned_free.size(); ++i)
            if (wr->pinned_free[i].second >= j.bytes) {
                j.host = wr->pinned_free[i].first; j.cap = wr->pinned_free[i].second;
                wr->pinned_free.erase(wr->pinned_free.begin() + i);
                break;
            }
    }
    if (!j.host) {
        P3D_CUDA_TRY(cudaMallocHost((void**)&j.host, j.bytes));
        j.cap = j.bytes;
    }
    P3D_CUDA_TRY(cudaGetDevice(&j.device));
    for (size_t i = 0, o = 0; i < (size_t)n; o += bytes[i++])
        P3D_CUDA_TRY(cudaMemcpyAsync(j.host + o, src[i], bytes[i], cudaMemcpyDeviceToHost, stream));
    P3D_CUDA_TRY(cudaEventCreateWithFlags(&j.ev, cudaEventDisableTiming | cudaEventBlockingSync));
    P3D_CUDA_TRY(cudaEventRecord(j.ev, stream));
    {
        std::lock_guard<std::mutex> lk(wr->m);
        wr->q.push_back(std::move(j));
        ++wr->inflight;
    }
    wr->cv_work.notify_one();
    return P3D_OK;
}

}  // namespace
}  // namespace p3d

extern "C" int p3d_png_writer_submit(void* writer, const uint8_t* dev_scanlines, int32_t h, int32_t w, int32_t channels,
                                     const char* path, void* stream) {
    if (int rc = check_image(writer, dev_scanlines, h, w, channels, path)) return rc;
    Job j;
    j.path = path; j.h = h; j.w = w; j.c = channels;
    const void* src[1] = {dev_scanlines};
    const size_t bytes[1] = {p3d_png_scanline_bytes(h, w, channels)};
    return submit_device((Writer*)writer, j, src, bytes, 1, (cudaStream_t)stream);
}

extern "C" int p3d_png_writer_submit_encoded(void* writer, const uint8_t* dev_file, const uint64_t* dev_len, int32_t h, int32_t w,
                                             int32_t channels, const char* path, void* stream) {
    if (int rc = check_image(writer, dev_file, h, w, channels, path)) return rc;
    P3D_REQUIRE(dev_len != nullptr, "p3d_png_writer_submit_encoded: NULL length pointer");
    const size_t bound = p3d_png_device_bound(h, w, channels);
    P3D_REQUIRE(bound != 0, "p3d_png_writer_submit_encoded: h=%d w=%d c=%d outside the device encoder's envelope", h, w, channels);
    Job j;
    j.path = path; j.h = h; j.w = w; j.c = channels; j.encoded = true;
    const void* src[2] = {dev_len, dev_file};
    const size_t bytes[2] = {sizeof(uint64_t), bound};
    return submit_device((Writer*)writer, j, src, bytes, 2, (cudaStream_t)stream);
}

extern "C" int p3d_png_writer_submit_host(void* writer, const uint8_t* host_scanlines, int32_t h, int32_t w, int32_t channels,
                                          const char* path) {
    if (int rc = check_image(writer, host_scanlines, h, w, channels, path)) return rc;
    Writer* wr = (Writer*)writer;
    Job j;
    j.path = path; j.h = h; j.w = w; j.c = channels; j.bytes = j.cap = p3d_png_scanline_bytes(h, w, channels); j.pinned = false; j.ev = nullptr; j.device = 0;
    j.host = (unsigned char*)malloc(j.bytes);
    P3D_REQUIRE(j.host != nullptr, "p3d_png_writer_submit_host: out of memory (%zu bytes)", j.bytes);
    memcpy(j.host, host_scanlines, j.bytes);
    {
        std::lock_guard<std::mutex> lk(wr->m);
        wr->q.push_back(std::move(j));
        ++wr->inflight;
    }
    wr->cv_work.notify_one();
    return P3D_OK;
}

extern "C" int p3d_png_writer_flush(void* writer, int32_t* n_failed) {
    P3D_REQUIRE(writer != nullptr, "p3d_png_writer_flush: NULL writer");
    Writer* wr = (Writer*)writer;
    std::unique_lock<std::mutex> lk(wr->m);
    wr->cv_done.wait(lk, [&] { return wr->inflight == 0; });
    if (n_failed) *n_failed = wr->failed;
    if (wr->failed) set_error("%s (%d image(s) failed)", wr->first_error.c_str(), wr->failed);
    const int failed = wr->failed;
    wr->failed = 0;
    wr->first_error.clear();
    return failed ? P3D_EINVAL : P3D_OK;
}

extern "C" int p3d_png_writer_destroy(void* writer) {
    P3D_REQUIRE(writer != nullptr, "p3d_png_writer_destroy: NULL writer");
    Writer* wr = (Writer*)writer;
    {
        std::unique_lock<std::mutex> lk(wr->m);
        wr->cv_done.wait(lk, [&] { return wr->inflight == 0; });
        wr->stop = true;
    }
    wr->cv_work.notify_all();
    for (auto& t : wr->threads) t.join();
    for (auto& b : wr->pinned_free) cudaFreeHost(b.first);
    delete wr;
    return P3D_OK;
}
