/*
 * p3d_imageio.h - C ABI of the image output path behind the renderer (SURVEY.md 8f-4) and of the PNG input path of
 * the training set (load_images, at the end of this header).
 *
 * The reference's eval sweep ends every view with `I(out['image']).save(fn)` and `I(xyza).save(fn)`
 * (/root/reference/_scripts/eval/generate.py:141-148): a blocking `.cpu()` of fp32 images, torchvision's
 * `to_pil_image` (clamp to [0,1], x255, truncate to uint8: /root/reference/_util/twodee_v1.py:174-185) and PIL's PNG
 * encoder, all on the one Python thread that also drives the GPU.  Here
 *   - quantisation, channel interleave and PNG scan-line filtering (the five PNG filters + libpng's minimum-sum
 *     heuristic) run on the device: a view leaves the GPU as 0.79 MB of filtered bytes instead of 3.1 MB of fp32;
 *   - the copy to pinned host memory is asynchronous on the caller's stream, and a pool of host threads deflates
 *     (zlib) and writes the files, so rank 0's render loop never waits for an encoder.
 * Files are PNGs any decoder reads; the decoded PIXELS equal what the reference's `I(...).save` writes (the byte
 * stream differs: filter choice and deflate level are not part of the image).
 *
 * Return codes / p3d_last_error() as in p3d_render.h.
 */
#ifndef P3D_IMAGEIO_H_
#define P3D_IMAGEIO_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* Bytes of the filtered scan-line stream of one h x w image with `channels` 8-bit channels: h * (1 + w * channels). */
size_t p3d_png_scanline_bytes(int32_t h, int32_t w, int32_t channels);

/* fp32 images (N,C,H,W), C in {1,3,4} -> N filtered scan-line streams (device memory, N * p3d_png_scanline_bytes).
   value = clamp((x + shift[c]) * scale[c], 0, 1) * 255 truncated to uint8 - `I(t).pil()` for a float tensor
   (twodee_v1.py:184) with an optional per-channel affine in front (scale/shift: HOST arrays of c floats, read before the launch; NULL = identity), which is how the
   `xyza` image `cat([(xyz + bw/2)/bw, weights])` (generate.py:141-144) is produced without materialising it:
   pass `image` = xyz planes, `extra` = the weights plane.
     extra : optional (N,1,H,W) plane appended as the LAST channel (then C counts it: C-1 planes come from `image`). */
int p3d_image_to_png_scanlines(const float* image, const float* extra, int32_t n, int32_t c, int32_t h, int32_t w,
                               const float* scale, const float* shift, uint8_t* scanlines, void* stream);

/* Same quantisation, plain interleaved pixels (N,H,W,C) uint8 (no filter bytes) for consumers that want the array. */
int p3d_image_to_u8(const float* image, const float* extra, int32_t n, int32_t c, int32_t h, int32_t w,
                    const float* scale, const float* shift, uint8_t* out_nhwc, void* stream);

/* Synchronous host-side encoder: filtered scan-lines (host memory) -> a complete PNG file image in `out`.
   Returns P3D_EWORKSPACE (and sets *out_len to the needed size) when `cap` is too small; cap >= p3d_png_encode_bound
   always suffices.  No CUDA involved: usable (and tested) without a GPU. */
size_t p3d_png_encode_bound(int32_t h, int32_t w, int32_t channels);
int p3d_png_encode_host(const uint8_t* scanlines, int32_t h, int32_t w, int32_t channels, int32_t level,
                        uint8_t* out, size_t cap, size_t* out_len);

/* Asynchronous writer: a pool of `n_threads` host threads that deflate and write PNG files.
   compress_level: zlib 0..9 (PIL's default is 6; 1-3 keeps a 512^2 RGB image under ~5 ms of one core). */
int p3d_png_writer_create(int32_t n_threads, int32_t compress_level, void** writer);
/* Enqueue one image whose filtered scan-lines live in DEVICE memory: the D2H copy (into pinned staging owned by the
   writer) is enqueued on `stream` and the call returns at once; a worker waits for the copy, encodes and writes
   `path` (written as path + ".tmp" and renamed, so a reader never sees a partial file). */
int p3d_png_writer_submit(void* writer, const uint8_t* dev_scanlines, int32_t h, int32_t w, int32_t channels,
                          const char* path, void* stream);
/* Same with scan-lines already in HOST memory (copied before the call returns).  No CUDA involved. */
int p3d_png_writer_submit_host(void* writer, const uint8_t* host_scanlines, int32_t h, int32_t w, int32_t channels,
                               const char* path);
/* Device encoder: N filtered scan-line streams (device memory, what p3d_image_to_png_scanlines writes) -> N complete PNG
   files in device memory (signature, IHDR, one IDAT with one zlib stream, IEND), deflated on the GPU: 16 KB segments of
   each stream are LZ77-matched (32 KB window, reaching back across segments) and coded as the smallest of a dynamic,
   fixed or stored block, then joined by sync flushes; every CRC-32, the Adler-32 and each file's length are computed on
   the device.  The bytes written are a function of the input bytes alone (not of the grid, the SM count or timing).
   Envelope: 1 <= n <= 65535, C in {1, 3, 4}, h, w >= 1 and h * (1 + w * C) <= 2^28; outside it the size queries return
   0 and the encoder P3D_EINVAL.
     bound       worst-case file bytes: 63 + h * (1 + w * C) + 10 * ceil(h * (1 + w * C) / 16384) (all-stored blocks).
     workspace   device scratch of p3d_png_device_workspace_bytes(n, h, w, C) bytes; its contents on entry do not matter.
     out         file i at out + i * out_stride (out_stride >= bound); bytes past its length are left untouched.
     out_lens    device array of n lengths, written by the encoder.
   Asynchronous on `stream`; P3D_EWORKSPACE when workspace_bytes is short, P3D_EINVAL on NULL pointers or bad shapes. */
size_t p3d_png_device_bound(int32_t h, int32_t w, int32_t channels);
size_t p3d_png_device_workspace_bytes(int32_t n, int32_t h, int32_t w, int32_t channels);
int p3d_png_encode_device(const uint8_t* scanlines, int32_t n, int32_t h, int32_t w, int32_t channels, void* workspace,
                          size_t workspace_bytes, uint8_t* out, size_t out_stride, uint64_t* out_lens, void* stream);
/* Enqueue one file that p3d_png_encode_device left in DEVICE memory: the D2H copies of its length and of
   p3d_png_device_bound(h, w, channels) bytes (into the writer's pinned staging) are enqueued on `stream` and the call
   returns at once; a worker waits for them and writes the file's length in bytes to `path` (".tmp" + rename, as above).
   The shape only sizes the copy: the worker writes what the device encoded. */
int p3d_png_writer_submit_encoded(void* writer, const uint8_t* dev_file, const uint64_t* dev_len, int32_t h, int32_t w,
                                  int32_t channels, const char* path, void* stream);
/* Wait until every submitted image is on disk; *n_failed = number of images that could not be written since the
   last flush (p3d_last_error() has the first failure's message). */
int p3d_png_writer_flush(void* writer, int32_t* n_failed);
int p3d_png_writer_destroy(void* writer);

/* ---- Image input: PNG files decoded on the device (DESIGN.md 4.7) ----
   The training set's chain `I(path).resize(size)[.convert('RGBA').bg('w').convert('RGB')].t()` (twodee_v1.py) for a
   batch of files: the host inspects each file and packs its zlib stream, the device inflates, unfilters, resizes
   (PIL's nearest), optionally composites onto white (PIL's integer `Image.alpha_composite`) and writes float32 / 255.
   Supported: colour type 0 at 8 bits (PIL mode L), types 2 and 6 at 8 or 16 bits (RGB / RGBA; PIL keeps the high byte
   of a 16-bit sample), compression 0, filter method 0, no interlace, and no tRNS chunk on type 0 or 2. */
typedef struct {
    int32_t h, w;
    int32_t channels;       /* colour type 0 / 2 / 6 -> 1 / 3 / 4 */
    int32_t depth;          /* bits per sample: 8, or 16 for 3 and 4 channels */
    int32_t n_idat;         /* IDAT chunks, zero-length ones included */
    int32_t reserved;
    uint64_t stream_bytes;  /* the zlib stream: every IDAT payload, concatenated */
} p3d_png_info;

/* Inspect one PNG file in host memory (`len` bytes): the signature, every chunk's length and CRC, IHDR, consecutive
   IDATs and IEND; ancillary chunks are skipped and unknown critical chunks refused.  Anything outside the supported set
   is refused with P3D_EINVAL and a message naming the field.  When `stream` is not NULL the IDAT payloads are copied
   there, info->stream_bytes of them.  No CUDA involved. */
int p3d_png_inspect(const uint8_t* file, size_t len, p3d_png_info* info, uint8_t* stream);

/* One image of a device decode.  The job array lives in device memory. */
typedef struct {
    uint64_t in_offset, in_bytes;  /* its zlib stream: in[in_offset, in_offset + in_bytes) */
    uint64_t ws_offset;            /* its workspace span: 16-byte aligned, p3d_png_decode_workspace_bytes(...) bytes */
    int32_t h, w, channels, depth; /* from p3d_png_inspect */
    int32_t slot;                  /* output image: out + slot * out_channels * out_h * out_w; distinct per job */
    int32_t reserved;
} p3d_png_decode_job;

/* Per-image status codes written by p3d_png_decode_device (and returned by p3d_png_inflate_host). */
#define P3D_PNG_OK          0
#define P3D_PNG_EJOB        1   /* the job's spans leave the buffers, or its fields leave the envelope */
#define P3D_PNG_EHEADER     2   /* zlib header: method other than 8, CINFO above 7, bad FCHECK, or a preset dictionary */
#define P3D_PNG_EBLOCK      3   /* block type 3, or a stored block whose LEN and NLEN disagree */
#define P3D_PNG_ECODES      4   /* dynamic block header: too many symbols, bad repeat, over-subscribed or incomplete
                                   code lengths, or no end-of-block code */
#define P3D_PNG_ESYMBOL     5   /* bits that are no code of the block, literal/length 286-287 or distance 30-31 */
#define P3D_PNG_EDISTANCE   6   /* a match reaching back past the start of the output */
#define P3D_PNG_ELONG       7   /* more output than h * (1 + w * bytes per pixel) */
#define P3D_PNG_ESHORT      8   /* less output than that */
#define P3D_PNG_ETRUNCATED  9   /* the input ends before the stream (or its Adler-32) does */
#define P3D_PNG_EADLER     10   /* the Adler-32 trailer does not match the output */
#define P3D_PNG_EFILTER    11   /* a scan-line filter byte above 4 */

/* Device workspace of one image decoded to out_h x out_w: its decompressed bytes h * (1 + w * channels * depth / 8),
   16-byte aligned, then out_w + out_h int32 resize indices.  0 outside the envelope: h, w >= 1, a supported
   (channels, depth), h * (1 + w * channels * depth / 8) <= 2^28 and 1 <= out_h, out_w <= 32768. */
size_t p3d_png_decode_workspace_bytes(int32_t h, int32_t w, int32_t channels, int32_t depth, int32_t out_h, int32_t out_w);

/* Decode n images (1 <= n <= 65535): `in` (device, in_bytes) holds the packed zlib streams, `jobs` (device, n) say
   where each is and where it goes.  out (device, float32) is (n, out_channels, out_h, out_w); out_channels is 3 when
   white_background is set, else every job's channel count.  status (device, n int32) gets one P3D_PNG_* code per job;
   a job with a non-zero code has its output image zeroed (when its slot is valid) and touches nothing outside its own
   spans, and the other jobs decode exactly as they would alone.  Every job is checked against in_bytes and
   workspace_bytes on the device.  Asynchronous on `stream` (three kernels); P3D_EINVAL on NULL pointers or a batch
   outside the envelope.  The output is a function of the input bytes alone. */
int p3d_png_decode_device(const uint8_t* in, size_t in_bytes, const p3d_png_decode_job* jobs, int32_t n, int32_t out_h,
                          int32_t out_w, int32_t out_channels, int32_t white_background, void* workspace,
                          size_t workspace_bytes, float* out, int32_t* status, void* stream);

/* The device decoder's inflate (bit reader, Huffman tables, copies, Adler-32) run on the CPU, for tests and debugging
   of malformed streams; not an image path.  Returns the P3D_PNG_* status of inflating the zlib stream into exactly
   raw_len bytes (1 <= raw_len <= 2^28), or P3D_EINVAL on NULL pointers. */
int p3d_png_inflate_host(const uint8_t* stream, size_t len, uint8_t* raw, size_t raw_len);

#ifdef __cplusplus
}
#endif
#endif /* P3D_IMAGEIO_H_ */
