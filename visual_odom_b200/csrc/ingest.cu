// ingest.cu -- image ingest (SURVEY.md 8f row N3): what the reference's loadImageLeft / loadImageRight do per frame
// (reference src/utils.cpp:172-190: cv::imread(IMREAD_COLOR) of <seq>/image_0/%06d.png, <seq>/image_1/%06d.png,
// then cv::cvtColor(BGR2GRAY)), re-designed for a GPU consumer:
//
//   * a small PNG decoder (zlib inflate + scanline un-filtering, non-interlaced, every colour type / bit depth) that
//     writes what imread(IMREAD_COLOR) + cvtColor would: BGR and/or the 15-bit fixed-point gray
//     (b*3735 + g*19235 + r*9798 + 2^14) >> 15 -- identical to OpenCV 4.13, checked over the whole colour cube in
//     tests/test_ingest.py.  Inflate is a serial Huffman stream per image, so it stays on host threads; one image is
//     ~0.5 MB, so the parallelism is ACROSS images, not inside one;
//   * a prefetching sequence reader: worker threads decode frames ahead of the consumer straight into a ring of
//     PINNED buffers, so vo_seq_push's H2D copy is a single async DMA and never waits for the file system;
//   * for colour sources the BGR bytes go to the device as they are and k_bgr_to_gray converts them there (inside the
//     frame's CUDA graph); gray sources (KITTI) need no conversion at all (the formula is the identity on b=g=r);
//   * images already in device memory (vo_dimage: gray, interleaved or planar BGR / RGB, any pitch and alignment) are
//     read by the same kernel straight into the raw gray planes (vo_seq_*_device, vo_batch_submit_device).
#include "ctx.h"
#include "remap_math.cuh"
#include <zlib.h>
#include <atomic>
#include <condition_variable>
#include <cstdio>
#include <cstring>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

// ------------------------------------------------------------------------------------------------ PNG
namespace {

struct PngHeader { uint32_t w = 0, h = 0; int depth = 0, ctype = 0, interlace = 0; };

inline uint32_t be32(const uint8_t* p) { return ((uint32_t)p[0] << 24) | ((uint32_t)p[1] << 16) | ((uint32_t)p[2] << 8) | p[3]; }
inline int samples_of(int ctype) { return ctype == 0 ? 1 : ctype == 2 ? 3 : ctype == 3 ? 1 : ctype == 4 ? 2 : ctype == 6 ? 4 : 0; }
inline uint8_t gray_of(int b, int g, int r) { return (uint8_t)((b * 3735 + g * 19235 + r * 9798 + (1 << 14)) >> 15); }

int png_header(const uint8_t* d, size_t n, PngHeader& hd, std::string& err)
{
    static const uint8_t sig[8] = {0x89, 'P', 'N', 'G', 0x0d, 0x0a, 0x1a, 0x0a};
    if (n < 8 + 25 || memcmp(d, sig, 8) != 0) { err = "not a PNG file"; return VO_E_INVALID; }
    if (be32(d + 8) != 13 || memcmp(d + 12, "IHDR", 4) != 0) { err = "PNG: IHDR is not the first chunk"; return VO_E_INVALID; }
    const uint8_t* p = d + 16;
    hd.w = be32(p); hd.h = be32(p + 4); hd.depth = p[8]; hd.ctype = p[9]; hd.interlace = p[12];
    if (hd.w == 0 || hd.h == 0 || hd.w > (1u << 16) || hd.h > (1u << 16)) { err = "PNG: unreasonable size"; return VO_E_INVALID; }
    if (p[10] != 0 || p[11] != 0) { err = "PNG: unknown compression / filter method"; return VO_E_INVALID; }
    const int ns = samples_of(hd.ctype);
    bool ok = ns != 0;
    if (hd.ctype == 0) ok = ok && (hd.depth == 1 || hd.depth == 2 || hd.depth == 4 || hd.depth == 8 || hd.depth == 16);
    else if (hd.ctype == 3) ok = ok && (hd.depth == 1 || hd.depth == 2 || hd.depth == 4 || hd.depth == 8);
    else ok = ok && (hd.depth == 8 || hd.depth == 16);
    if (!ok) { err = "PNG: invalid colour type / bit depth"; return VO_E_INVALID; }
    if (hd.interlace != 0) { err = "PNG: Adam7 interlacing is not supported"; return VO_E_UNSUPPORTED; }
    return VO_OK;
}

inline int paeth(int a, int b, int c)
{
    const int p = a + b - c, pa = abs(p - a), pb = abs(p - b), pc = abs(p - c);
    return (pa <= pb && pa <= pc) ? a : (pb <= pc ? b : c);
}

// undo the per-scanline filters in place; `raw` holds h x (1 + rowbytes)
int png_unfilter(uint8_t* raw, size_t rowbytes, uint32_t h, int bpp, std::string& err)
{
    const uint8_t* prev = nullptr;
    for (uint32_t y = 0; y < h; y++) {
        uint8_t* row = raw + (size_t)y * (rowbytes + 1);
        const int ft = row[0];
        uint8_t* x = row + 1;
        switch (ft) {
        case 0: break;
        case 1:
            for (size_t i = bpp; i < rowbytes; i++) x[i] = (uint8_t)(x[i] + x[i - bpp]);
            break;
        case 2:
            if (prev) for (size_t i = 0; i < rowbytes; i++) x[i] = (uint8_t)(x[i] + prev[i]);
            break;
        case 3:
            for (size_t i = 0; i < rowbytes; i++) {
                const int a = i >= (size_t)bpp ? x[i - bpp] : 0, b = prev ? prev[i] : 0;
                x[i] = (uint8_t)(x[i] + ((a + b) >> 1));
            }
            break;
        case 4:
            for (size_t i = 0; i < rowbytes; i++) {
                const int a = i >= (size_t)bpp ? x[i - bpp] : 0, b = prev ? prev[i] : 0, c = (prev && i >= (size_t)bpp) ? prev[i - bpp] : 0;
                x[i] = (uint8_t)(x[i] + paeth(a, b, c));
            }
            break;
        default:
            err = "PNG: bad scanline filter type"; return VO_E_INVALID;
        }
        prev = x;
    }
    return VO_OK;
}

// file bytes -> BGR (3 B/px) and/or gray (1 B/px); either output may be null
int png_decode(const uint8_t* d, size_t n, uint8_t* bgr, size_t bgr_pitch, uint8_t* gray, size_t gray_pitch,
               std::vector<uint8_t>& idat, std::vector<uint8_t>& raw, std::string& err)
{
    PngHeader hd;
    int rc = png_header(d, n, hd, err);
    if (rc) return rc;
    uint8_t plte[768];
    int nplte = 0;
    idat.clear();
    size_t pos = 8;
    bool end = false;
    while (!end) {
        if (pos + 12 > n) { err = "PNG: truncated file"; return VO_E_INVALID; }
        const uint32_t len = be32(d + pos);
        if ((size_t)len > n - pos - 12) { err = "PNG: truncated chunk"; return VO_E_INVALID; }
        const uint8_t* type = d + pos + 4;
        const uint8_t* data = d + pos + 8;
        if ((uint32_t)crc32(crc32(0L, type, 4), data, len) != be32(data + len)) { err = "PNG: chunk CRC mismatch"; return VO_E_INVALID; }
        if (!memcmp(type, "IDAT", 4)) idat.insert(idat.end(), data, data + len);
        else if (!memcmp(type, "PLTE", 4)) { nplte = (int)(len / 3 < 256 ? len / 3 : 256); memcpy(plte, data, (size_t)nplte * 3); }
        else if (!memcmp(type, "IEND", 4)) end = true;
        pos += 12 + (size_t)len;
    }
    if (hd.ctype == 3 && nplte == 0) { err = "PNG: palette image without PLTE"; return VO_E_INVALID; }
    const int ns = samples_of(hd.ctype), bits = ns * hd.depth;
    const size_t rowbytes = ((size_t)hd.w * bits + 7) / 8;
    const int bpp = bits >= 8 ? bits / 8 : 1;
    raw.resize((size_t)hd.h * (rowbytes + 1));
    {
        z_stream zs;
        memset(&zs, 0, sizeof(zs));
        if (inflateInit(&zs) != Z_OK) { err = "zlib: inflateInit failed"; return VO_E_INVALID; }
        zs.next_in = idat.data(); zs.avail_in = (uInt)idat.size();
        zs.next_out = raw.data(); zs.avail_out = (uInt)raw.size();
        const int zr = inflate(&zs, Z_FINISH);
        const size_t got = raw.size() - zs.avail_out;
        inflateEnd(&zs);
        if ((zr != Z_STREAM_END && zr != Z_OK && zr != Z_BUF_ERROR) || got != raw.size()) { err = "PNG: corrupt or short image data"; return VO_E_INVALID; }
    }
    if ((rc = png_unfilter(raw.data(), rowbytes, hd.h, bpp, err))) return rc;

    const int step = hd.depth == 16 ? 2 : 1;          // 16-bit samples: the high byte (what imread's 8-bit output keeps)
    for (uint32_t y = 0; y < hd.h; y++) {
        const uint8_t* x = raw.data() + (size_t)y * (rowbytes + 1) + 1;
        uint8_t* ob = bgr ? bgr + (size_t)y * bgr_pitch : nullptr;
        uint8_t* og = gray ? gray + (size_t)y * gray_pitch : nullptr;
        for (uint32_t i = 0; i < hd.w; i++) {
            int r, g, b;
            if (hd.ctype == 2 || hd.ctype == 6) {
                const uint8_t* s = x + (size_t)i * ns * step;
                r = s[0]; g = s[step]; b = s[2 * step];
            } else {
                int v;
                if (hd.depth >= 8) v = x[(size_t)i * ns * step];
                else {
                    const int per = 8 / hd.depth, sh = 8 - hd.depth * (1 + (int)(i % per));
                    v = (x[i / per] >> sh) & ((1 << hd.depth) - 1);
                    if (hd.ctype == 0) v = v * 255 / ((1 << hd.depth) - 1);
                }
                if (hd.ctype == 3) {
                    if (v >= nplte) { r = g = b = 0; }
                    else { r = plte[3 * v]; g = plte[3 * v + 1]; b = plte[3 * v + 2]; }
                } else r = g = b = v;
            }
            if (ob) { ob[3 * i] = (uint8_t)b; ob[3 * i + 1] = (uint8_t)g; ob[3 * i + 2] = (uint8_t)r; }
            if (og) og[i] = gray_of(b, g, r);
        }
    }
    return VO_OK;
}

int read_file(const std::string& path, std::vector<uint8_t>& out, std::string& err)
{
    FILE* f = fopen(path.c_str(), "rb");
    if (!f) { err = "cannot open " + path; return VO_E_INVALID; }
    fseek(f, 0, SEEK_END);
    const long sz = ftell(f);
    fseek(f, 0, SEEK_SET);
    if (sz <= 0) { fclose(f); err = "empty file " + path; return VO_E_INVALID; }
    out.resize((size_t)sz);
    const size_t got = fread(out.data(), 1, (size_t)sz, f);
    fclose(f);
    if (got != (size_t)sz) { err = "short read on " + path; return VO_E_INVALID; }
    return VO_OK;
}

thread_local std::string g_png_err;

}  // namespace

extern "C" const char* vo_png_last_error(void) { return g_png_err.c_str(); }

extern "C" int vo_png_info(const uint8_t* file_bytes, size_t n, int* w, int* h, int* color_type, int* bit_depth)
{
    PngHeader hd;
    g_png_err.clear();
    if (!file_bytes) { g_png_err = "null buffer"; return VO_E_INVALID; }
    const int rc = png_header(file_bytes, n, hd, g_png_err);
    if (rc) return rc;
    if (w) *w = (int)hd.w;
    if (h) *h = (int)hd.h;
    if (color_type) *color_type = hd.ctype;
    if (bit_depth) *bit_depth = hd.depth;
    return VO_OK;
}

extern "C" int vo_png_decode(const uint8_t* file_bytes, size_t n, uint8_t* bgr, size_t bgr_pitch, uint8_t* gray, size_t gray_pitch)
{
    g_png_err.clear();
    if (!file_bytes) { g_png_err = "null buffer"; return VO_E_INVALID; }
    std::vector<uint8_t> idat, raw;
    return png_decode(file_bytes, n, bgr, bgr_pitch, gray, gray_pitch, idat, raw, g_png_err);
}

// ------------------------------------------------------------------------------------------------ sequence reader
struct vo_reader {
    std::string dir;
    int first = 0, count = 0, depth = 0, w = 0, h = 0, channels = 1;
    size_t pitch = 0, img_bytes = 0;
    bool pinned = false;
    uint8_t* ring = nullptr;                        // depth x 2 images
    std::vector<int> state;                         // per frame: 0 = pending, 1 = decoded, -1 = failed
    std::vector<std::thread> workers;
    std::mutex mu;
    std::condition_variable cv_ready, cv_free;
    int next_claim = 0;                             // next frame a worker will take
    int consumed = 0;                               // frames handed out so far (the consumer may still use the last two)
    bool stop = false;
    std::string error;
    std::string frame_error;
};

static std::string frame_path(const std::string& dir, int cam, int frame_id)
{
    char name[64];
    snprintf(name, sizeof(name), "image_%d/%06d.png", cam, frame_id);          // utils.cpp:174,184
    std::string p = dir;
    if (!p.empty() && p.back() != '/') p += '/';
    return p + name;
}

static void reader_worker(vo_reader* rd)
{
    std::vector<uint8_t> file, idat, raw;
    for (;;) {
        int i;
        {
            std::unique_lock<std::mutex> lk(rd->mu);
            // frame i lives in slot i % depth; that slot is free once frame i - depth has been released, i.e. the
            // consumer has moved past it: it holds frame consumed-1 at most.
            // frame i lives in slot i % depth.  The consumer may still be using the last TWO frames it was handed
            // (frames consumed-1 and consumed-2: one being uploaded asynchronously while the next is requested), so
            // slot reuse needs i - depth < consumed - 2.
            rd->cv_free.wait(lk, [&] {
                const int c = rd->consumed > 2 ? rd->consumed : 2;
                return rd->stop || rd->next_claim >= rd->count || rd->next_claim < c + rd->depth - 2;
            });
            if (rd->stop || rd->next_claim >= rd->count) return;
            i = rd->next_claim++;
        }
        std::string err;
        int rc = VO_OK;
        for (int cam = 0; cam < 2 && rc == VO_OK; cam++) {
            uint8_t* dst = rd->ring + ((size_t)(i % rd->depth) * 2 + cam) * rd->img_bytes;
            rc = read_file(frame_path(rd->dir, cam, rd->first + i), file, err);
            if (rc) break;
            PngHeader hd;
            rc = png_header(file.data(), file.size(), hd, err);
            if (rc) break;
            if ((int)hd.w != rd->w || (int)hd.h != rd->h) { err = "image size changes inside the sequence"; rc = VO_E_INVALID; break; }
            if (rd->channels == 3) rc = png_decode(file.data(), file.size(), dst, rd->pitch, nullptr, 0, idat, raw, err);
            else rc = png_decode(file.data(), file.size(), nullptr, 0, dst, rd->pitch, idat, raw, err);
        }
        {
            std::lock_guard<std::mutex> lk(rd->mu);
            rd->state[i] = rc == VO_OK ? 1 : -1;
            if (rc != VO_OK && rd->frame_error.empty()) rd->frame_error = err;
        }
        rd->cv_ready.notify_all();
    }
}

extern "C" vo_reader* vo_reader_open(const char* sequence_dir, int first_frame, int n_frames, int threads, int depth, int force_channels)
{
    g_png_err.clear();
    if (!sequence_dir || n_frames <= 0 || first_frame < 0) { g_png_err = "vo_reader_open: bad argument"; return nullptr; }
    if (threads <= 0) threads = 4;
    if (depth < 3) depth = 3;
    vo_reader* rd = new vo_reader();
    rd->dir = sequence_dir; rd->first = first_frame; rd->count = n_frames; rd->depth = depth;
    std::vector<uint8_t> file;
    PngHeader hd;
    if (read_file(frame_path(rd->dir, 0, first_frame), file, g_png_err) || png_header(file.data(), file.size(), hd, g_png_err)) { delete rd; return nullptr; }
    rd->w = (int)hd.w; rd->h = (int)hd.h;
    // gray files (KITTI) are delivered as gray: imread(COLOR) replicates and cvtColor maps b=g=r=v back to v.
    // colour files are delivered as BGR and converted on the device (vo_seq_push_ex, channels = 3).
    rd->channels = force_channels == 1 || force_channels == 3 ? force_channels : ((hd.ctype == 0 || hd.ctype == 4) ? 1 : 3);
    rd->pitch = (size_t)rd->w * rd->channels;
    rd->img_bytes = (rd->pitch * rd->h + 255) & ~(size_t)255;
    const size_t total = rd->img_bytes * 2 * depth;
    void* p = nullptr;
    if (cudaHostAlloc(&p, total, cudaHostAllocDefault) == cudaSuccess) rd->pinned = true;
    else { cudaGetLastError(); p = malloc(total); }      // no CUDA device (CPU-only test box): plain host memory
    if (!p) { g_png_err = "vo_reader_open: out of memory"; delete rd; return nullptr; }
    rd->ring = (uint8_t*)p;
    rd->state.assign(n_frames, 0);
    for (int t = 0; t < threads; t++) rd->workers.emplace_back(reader_worker, rd);
    return rd;
}

extern "C" int vo_reader_next(vo_reader* rd, const uint8_t** left, const uint8_t** right, int* w, int* h, size_t* pitch,
                              int* channels, int* frame_id)
{
    if (!rd) return VO_E_INVALID;
    std::unique_lock<std::mutex> lk(rd->mu);
    if (rd->consumed >= rd->count) { rd->error = "vo_reader_next: end of sequence"; return VO_E_INVALID; }
    const int i = rd->consumed;
    rd->consumed++;                                 // releases the slot of frame i-2
    rd->cv_free.notify_all();
    rd->cv_ready.wait(lk, [&] { return rd->state[i] != 0; });
    if (rd->state[i] < 0) { rd->error = rd->frame_error; return VO_E_INVALID; }
    const uint8_t* base = rd->ring + (size_t)(i % rd->depth) * 2 * rd->img_bytes;
    if (left) *left = base;
    if (right) *right = base + rd->img_bytes;
    if (w) *w = rd->w;
    if (h) *h = rd->h;
    if (pitch) *pitch = rd->pitch;
    if (channels) *channels = rd->channels;
    if (frame_id) *frame_id = rd->first + i;
    return VO_OK;
}

extern "C" const char* vo_reader_error(vo_reader* rd) { return rd ? rd->error.c_str() : g_png_err.c_str(); }

extern "C" void vo_reader_close(vo_reader* rd)
{
    if (!rd) return;
    {
        std::lock_guard<std::mutex> lk(rd->mu);
        rd->stop = true;
    }
    rd->cv_free.notify_all();
    for (auto& t : rd->workers) t.join();
    if (rd->ring) { if (rd->pinned) cudaFreeHost(rd->ring); else free(rd->ring); }
    delete rd;
}

// ------------------------------------------------------------------------------------------------ device gray convert
// Source image -> raw gray plane (w bytes per row), 4 pixels per thread, 32-bit stores where the destination allows.
// Image z of the launch is tab[z] (caller device images: descriptors staged per submission), or, with tab == nullptr,
// `packed` advanced by z * packed_stride (the packed BGR staging of host colour input, whose graph-captured launch
// cannot take a per-frame table).  Sources may have any alignment, pitch and strides: every pixel is read with byte
// loads.  Colour: cv::cvtColor(BGR2GRAY / RGB2GRAY)'s fixed point; gray: the identity (which the formula is on b=g=r).
// With a geometry table (geo[img]: images of several sizes, w x h the envelope) image z is geo[z]'s own size, its packed
// source rows 3 * w[0] bytes apart (a table source keeps its own pitch) and its gray rows w[0].  A table entry with
// data == NULL (a retired or empty slot of the multi-sequence mode) is skipped: its plane keeps what it held.
__global__ void k_bgr_to_gray(const vo_dimage* __restrict__ tab, vo_dimage packed, size_t packed_stride, uint8_t* __restrict__ gray,
                              size_t img_stride_out, int w, int h, const PlaneGeom* __restrict__ geo, const RectMap* __restrict__ maps)
{
    const int img = blockIdx.z, y = blockIdx.y;
    const int x0 = 4 * (blockIdx.x * blockDim.x + threadIdx.x);
    vo_dimage src = packed;
    if (geo) { w = geo[img].w[0]; h = geo[img].h[0]; src.row_pitch = (size_t)3 * w; }
    if (x0 >= w || y >= h) return;
    if (tab) {
        src = tab[img];
        if (!src.data) return;
    } else src.data += (size_t)img * packed_stride;
    const size_t cs = src.channel_stride;
    // the gray value of source pixel (x, y)
    auto px = [&](int x, int yy) -> int {
        const uint8_t* p = src.data + (size_t)yy * src.row_pitch + (size_t)x * src.pixel_stride;
        if (src.format == VO_FMT_GRAY) return p[0];
        const int c0 = p[0], g = p[cs], c2 = p[2 * cs];
        return src.format == VO_FMT_RGB ? vorect::gray_of(c2, g, c0) : vorect::gray_of(c0, g, c2);
    };
    const RectMap m = maps ? maps[img] : RectMap{nullptr, nullptr};
    uint8_t* d = gray + (size_t)img * img_stride_out + (size_t)y * w + x0;
    uint8_t o[4];
#pragma unroll
    for (int i = 0; i < 4; i++) {
        if (x0 + i >= w) o[i] = 0;
        else if (m.xy) {            // cv::remap(INTER_LINEAR, BORDER_CONSTANT 0) of the converted image
            const size_t k = (size_t)y * w + x0 + i;
            o[i] = vorect::remap_pixel(m.xy[k], m.a[k], w, h, px);
        } else o[i] = (uint8_t)px(x0 + i, y);
    }
    if (x0 + 3 < w && ((size_t)(d - gray) & 3) == 0 && (((size_t)gray) & 3) == 0)
        *reinterpret_cast<uint32_t*>(d) = o[0] | (o[1] << 8) | (o[2] << 16) | ((uint32_t)o[3] << 24);
    else
        for (int i = 0; i < 4 && x0 + i < w; i++) d[i] = o[i];
}

int vo_launch_bgr_to_gray(const vo_dimage* d_tab, const vo_dimage& packed, size_t packed_stride, uint8_t* d_gray, size_t img_stride_out,
                          int w, int h, int n_img, cudaStream_t s, const PlaneGeom* geo, const RectMap* maps)
{
    dim3 grid(((w + 3) / 4 + 127) / 128, h, n_img);
    k_bgr_to_gray<<<grid, 128, 0, s>>>(d_tab, packed, packed_stride, d_gray, img_stride_out, w, h, geo, maps);
    return 1;
}

vo_dimage vo_packed_bgr(const uint8_t* d_bgr, int w)
{
    vo_dimage a;
    a.data = d_bgr; a.row_pitch = (size_t)3 * w; a.pixel_stride = 3; a.channel_stride = 1; a.format = VO_FMT_BGR;
    return a;
}

int vo_check_dimage(vo_ctx* ctx, const char* who, const char* name, const vo_dimage* im, int w)
{
    if (!im || !im->data) { vo_set_error(ctx, "%s: %s: null image", who, name); return VO_E_INVALID; }
    if (im->format != VO_FMT_GRAY && im->format != VO_FMT_BGR && im->format != VO_FMT_RGB) {
        vo_set_error(ctx, "%s: %s: unknown format %d (VO_FMT_GRAY, VO_FMT_BGR or VO_FMT_RGB)", who, name, im->format);
        return VO_E_INVALID;
    }
    if (im->pixel_stride < 1) { vo_set_error(ctx, "%s: %s: pixel_stride %d < 1", who, name, im->pixel_stride); return VO_E_INVALID; }
    if (im->row_pitch < (size_t)w * im->pixel_stride) {
        vo_set_error(ctx, "%s: %s: row_pitch %zu < %d pixels x pixel_stride %d", who, name, im->row_pitch, w, im->pixel_stride);
        return VO_E_INVALID;
    }
    if (im->format != VO_FMT_GRAY && im->channel_stride < 1) { vo_set_error(ctx, "%s: %s: channel_stride 0 for a colour image", who, name); return VO_E_INVALID; }
    VO_CUDA_CHECK(cudaSetDevice(ctx->device));
    cudaPointerAttributes a;
    const cudaError_t e = cudaPointerGetAttributes(&a, im->data);
    if (e != cudaSuccess) { cudaGetLastError(); vo_set_error(ctx, "%s: %s: not a CUDA pointer (%s)", who, name, cudaGetErrorString(e)); return VO_E_INVALID; }
    if (a.type == cudaMemoryTypeManaged) return VO_OK;
    if (a.type != cudaMemoryTypeDevice) {
        vo_set_error(ctx, "%s: %s is %s memory; the *_device entry points take device memory", who, name,
                     a.type == cudaMemoryTypeHost ? "pinned host" : "host");
        return VO_E_INVALID;
    }
    if (a.device != ctx->device) { vo_set_error(ctx, "%s: %s is on device %d, the context on device %d", who, name, a.device, ctx->device); return VO_E_INVALID; }
    return VO_OK;
}

int vo_ingest_device(vo_ctx* ctx, const vo_dimage* h_tab, int n, int plane0, cudaStream_t st, const PlaneGeom* geo,
                     const RectMap* h_maps)
{
    const size_t plane = (size_t)ctx->w * ctx->h;
    VO_CUDA_CHECK(cudaMemcpyAsync(ctx->d_ingest_tab + plane0, h_tab, (size_t)n * sizeof(vo_dimage), cudaMemcpyHostToDevice, st));
    if (h_maps)
        VO_CUDA_CHECK(cudaMemcpyAsync(ctx->d_ingest_map + plane0, h_maps, (size_t)n * sizeof(RectMap), cudaMemcpyHostToDevice, st));
    ctx->launches += vo_launch_bgr_to_gray(ctx->d_ingest_tab + plane0, vo_dimage{}, 0, ctx->d_raw + (size_t)plane0 * plane, plane,
                                           ctx->w, ctx->h, n, st, geo, h_maps ? ctx->d_ingest_map + plane0 : nullptr);
    VO_CUDA_CHECK(cudaGetLastError());
    return VO_OK;
}

int vo_ensure_bgr(vo_ctx* ctx, size_t bytes)
{
    if (ctx->bgr_bytes >= bytes) return VO_OK;
    if (ctx->d_bgr) cudaFree(ctx->d_bgr);
    ctx->d_bgr = nullptr; ctx->bgr_bytes = 0;
    vo_drop_graphs(ctx);                          // graphs hold the old pointer
    VO_CUDA_CHECK(cudaMalloc(&ctx->d_bgr, bytes));
    ctx->bgr_bytes = bytes;
    return VO_OK;
}

extern "C" int vo_bgr_to_gray(vo_ctx* ctx, const uint8_t* bgr, size_t pitch, int w, int h, uint8_t* gray, size_t gray_pitch)
{
    if (!ctx) return VO_E_INVALID;
    if (!bgr || !gray || w <= 0 || h <= 0 || pitch < (size_t)3 * w || gray_pitch < (size_t)w) { vo_set_error(ctx, "vo_bgr_to_gray: bad argument"); return VO_E_INVALID; }
    { int rcc = vo_claim_buffers(ctx, "vo_bgr_to_gray"); if (rcc) return rcc; }
    VO_CUDA_CHECK(cudaSetDevice(ctx->device));
    const size_t in_bytes = ((size_t)3 * w * h + 255) & ~(size_t)255;
    int rc = vo_ensure_bgr(ctx, in_bytes + (size_t)w * h);
    if (rc) return rc;
    uint8_t* d_in = ctx->d_bgr;
    uint8_t* d_out = ctx->d_bgr + in_bytes;
    VO_CUDA_CHECK(cudaMemcpy2DAsync(d_in, (size_t)3 * w, bgr, pitch, (size_t)3 * w, h, cudaMemcpyHostToDevice, ctx->stream));
    ctx->launches += vo_launch_bgr_to_gray(nullptr, vo_packed_bgr(d_in, w), 0, d_out, 0, w, h, 1, ctx->stream);
    VO_CUDA_CHECK(cudaGetLastError());
    VO_CUDA_CHECK(cudaMemcpy2DAsync(gray, gray_pitch, d_out, w, w, h, cudaMemcpyDeviceToHost, ctx->stream));
    VO_CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
    return VO_OK;
}
