// extern "C" surface of libsnn_b200.so for contexts, tensors, weights, single-operator launches and timers.
// (The whole-model engine entry points live in engine/model_capi.cpp.) See include/snnb.h for the reference
// interface each entry point replaces.
#include <algorithm>
#include <climits>
#include <cstdarg>
#include <cstdlib>
#include <cstring>
#include <memory>

#include "snnb_internal.h"

namespace snnb {

static thread_local char g_err[1024] = "";
void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}
const char* get_error() { return g_err; }

bool pdl_enabled() {
    static const bool on = getenv("SNNB_NO_PDL") == nullptr;
    return on;
}

int ensure_stage(snnb_context* ctx, size_t bytes) {
    if (ctx->stage_dev_bytes < bytes) {
        if (ctx->stage_dev) cudaFree(ctx->stage_dev);
        ctx->stage_dev       = nullptr;
        ctx->stage_dev_bytes = 0;
        SNNB_CUDA_OK(cudaMalloc(&ctx->stage_dev, bytes));
        ctx->stage_dev_bytes = bytes;
    }
    return 0;
}
static int ensure_stage_host(snnb_context* ctx, size_t bytes) {
    if (ctx->stage_host_bytes < bytes) {
        if (ctx->stage_host) cudaFreeHost(ctx->stage_host);
        ctx->stage_host       = nullptr;
        ctx->stage_host_bytes = 0;
        SNNB_CUDA_OK(cudaMallocHost(&ctx->stage_host, bytes));
        ctx->stage_host_bytes = bytes;
    }
    return 0;
}

int tensor_alloc(snnb_context* ctx, int n, int h, int w, int c, snnb_tensor** out, bool lo_plane) {
    SNNB_REQUIRE(ctx && out, "tensor_alloc: null argument");
    SNNB_REQUIRE(n > 0 && h > 0 && w > 0 && c > 0, "tensor_alloc: bad dims %d %d %d %d", n, h, w, c);
    auto t   = std::make_unique<snnb_tensor>();
    t->ctx   = ctx;
    t->n = n, t->h = h, t->w = w, t->c = c, t->cp = round_up(c, 8);
    size_t elems   = (size_t) n * h * w * t->cp;
    t->plane_elems = (elems + 63) / 64 * 64;
    const size_t planes = lo_plane ? 2 : 1; // half-precision storage mode: the hi plane alone
    SNNB_CUDA_OK(cudaMalloc(&t->hi, t->plane_elems * planes * sizeof(__half)));
    t->lo = lo_plane ? t->hi + t->plane_elems : nullptr;
    SNNB_CUDA_OK(cudaMemsetAsync(t->hi, 0, t->plane_elems * planes * sizeof(__half), ctx->stream));
    *out = t.release();
    return 0;
}

// The compact 4-channel copy a stride-2 RGB stem reads (snnb_tensor::feed_*): zeroed once, the input kernels only ever write
// the image area, so the margins stay the constant padding.
int tensor_alloc_feed(snnb_tensor* t, int feed_h, int feed_w, int py, int px) {
    SNNB_REQUIRE(t && !t->feed_hi && t->c <= 4 && feed_h >= t->h + py && feed_w >= t->w + px && (feed_w & 1) == 0 && (px & 1) == 0, "tensor_alloc_feed: bad argument");
    const size_t plane  = ((size_t) t->n * feed_h * feed_w * 4 + 63) / 64 * 64;
    const size_t planes = t->lo ? 2 : 1;
    SNNB_CUDA_OK(cudaMalloc(&t->feed_hi, plane * planes * sizeof(__half)));
    SNNB_CUDA_OK(cudaMemsetAsync(t->feed_hi, 0, plane * planes * sizeof(__half), t->ctx->stream));
    t->feed_lo = t->lo ? t->feed_hi + plane : nullptr;
    t->feed_h = feed_h, t->feed_w = feed_w, t->feed_py = py, t->feed_px = px;
    return 0;
}

} // namespace snnb

using namespace snnb;

#define CHECK_DIMS_EQ(a, b, what) SNNB_REQUIRE((a)->n == (b)->n && (a)->h == (b)->h && (a)->w == (b)->w && (a)->c == (b)->c, what ": tensor dims differ")

extern "C" {

int snnb_version(void) { return SNNB_VERSION; }
int snnb_context_set_precision(snnb_context* ctx, int precision) {
    SNNB_REQUIRE(ctx && (precision == SNNB_PRECISION_FP32X3 || precision == SNNB_PRECISION_FP16W), "snnb_context_set_precision: FP32X3 or FP16W (FP16 storage is a model option)");
    ctx->precision = precision;
    return 0;
}
const char* snnb_last_error(void) { return get_error(); }

int snnb_context_create(int device, snnb_context** out) {
    SNNB_REQUIRE(out, "snnb_context_create: null out");
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count == 0) {
        set_error("snnb_context_create: no CUDA device available (%s). This library has no CPU fallback.", cudaGetErrorString(e));
        return 1;
    }
    SNNB_REQUIRE(device >= 0 && device < count, "snnb_context_create: device %d out of range (%d devices)", device, count);
    SNNB_CUDA_OK(cudaSetDevice(device));
    cudaDeviceProp prop;
    SNNB_CUDA_OK(cudaGetDeviceProperties(&prop, device));
    SNNB_REQUIRE(prop.major == 9 && prop.minor == 0, "snnb_context_create: device %d is sm_%d%d; this library is built for sm_90a (H100) only", device, prop.major,
                 prop.minor);
    auto ctx      = std::make_unique<snnb_context>();
    ctx->device   = device;
    ctx->sm_count = prop.multiProcessorCount;
    SNNB_CUDA_OK(cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking));
    *out = ctx.release();
    return 0;
}

int snnb_context_destroy(snnb_context* ctx) {
    if (!ctx) return 0;
    cudaSetDevice(ctx->device);
    cudaStreamSynchronize(ctx->stream);
    if (ctx->stage_dev) cudaFree(ctx->stage_dev);
    if (ctx->stage_host) cudaFreeHost(ctx->stage_host);
    for (void* b : ctx->scratch_blocks) cudaFree(b);
    cudaStreamDestroy(ctx->stream);
    delete ctx;
    return 0;
}

int snnb_sync(snnb_context* ctx) {
    SNNB_REQUIRE(ctx, "snnb_sync: null context");
    SNNB_CUDA_OK(cudaStreamSynchronize(ctx->stream));
    return 0;
}
void* snnb_context_stream(snnb_context* ctx) { return ctx ? (void*) ctx->stream : nullptr; }
uint64_t snnb_launch_count(snnb_context* ctx) { return ctx ? ctx->launches : 0; }
int snnb_rois_from_detections(snnb_context* ctx, const float* rows_dev, const int* counts_dev, int num_frames, int max_rows, int frame_width, int frame_height,
                              const snnb_roi_select* sel, snnb_roi* rois_dev, int capacity, int* count_dev, void* stream) {
    SNNB_REQUIRE(ctx, "snnb_rois_from_detections: null context");
    SNNB_CUDA_OK(cudaSetDevice(ctx->device));
    return rois_from_detections(ctx, rows_dev, counts_dev, num_frames, max_rows, frame_width, frame_height, sel, rois_dev, capacity, count_dev,
                                static_cast<cudaStream_t>(stream));
}
int snnb_rois_from_detections_list(snnb_context* ctx, const float* rows_dev, const int* counts_dev, int num_frames, int max_rows, const int* frame_wh,
                                   const snnb_roi_select* sel, snnb_roi* rois_dev, int capacity, int* count_dev, void* stream) {
    SNNB_REQUIRE(ctx, "snnb_rois_from_detections_list: null context");
    SNNB_CUDA_OK(cudaSetDevice(ctx->device));
    return rois_from_detections_list(ctx, rows_dev, counts_dev, num_frames, max_rows, frame_wh, sel, rois_dev, capacity, count_dev, static_cast<cudaStream_t>(stream));
}
// Tile starts along one axis of `size` pixels for tiles of t <= size with at least `ov` < t pixels of overlap: n = 1 + ceil((size - t) /
// (t - ov)) tiles, tile i at i * (size - t) / (n - 1), so neighbours are at most t - ov apart and the last tile ends at size.
static long long tileCount(int size, int t, int ov) { return 1 + ((long long) size - t + (t - ov) - 1) / (t - ov); }
static int tileStart(int size, int t, long long n, long long i) { return n == 1 ? 0 : (int) (i * (size - t) / (n - 1)); }
int snnb_tile_rois(int frame, int frame_w, int frame_h, int tile_w, int tile_h, int min_overlap, snnb_roi* rois_host, int capacity, int* count) {
    SNNB_REQUIRE(count, "snnb_tile_rois: null count");
    SNNB_REQUIRE(frame_w >= 1 && frame_h >= 1, "snnb_tile_rois: frame size %d x %d; width and height must be >= 1", frame_w, frame_h);
    SNNB_REQUIRE(tile_w >= 1 && tile_h >= 1, "snnb_tile_rois: tile size %d x %d; width and height must be >= 1", tile_w, tile_h);
    const int tw = std::min(tile_w, frame_w), th = std::min(tile_h, frame_h);
    SNNB_REQUIRE(min_overlap >= 0 && min_overlap < std::min(tw, th), "snnb_tile_rois: min_overlap %d is outside 0..%d (the tile %d x %d, clamped to the frame)",
                 min_overlap, std::min(tw, th) - 1, tw, th);
    const long long nx = tileCount(frame_w, tw, min_overlap), ny = tileCount(frame_h, th, min_overlap), n = nx * ny;
    if (n > capacity) {
        *count = (int) std::min(n, (long long) INT_MAX);
        SNNB_REQUIRE(false, "snnb_tile_rois: %lld x %lld = %lld tiles; capacity %d", nx, ny, n, capacity);
    }
    SNNB_REQUIRE(rois_host, "snnb_tile_rois: null rois");
    for (long long j = 0; j < ny; ++j)
        for (long long i = 0; i < nx; ++i)
            rois_host[j * nx + i] = snnb_roi {frame, (int) (j * nx + i), tileStart(frame_w, tw, nx, i), tileStart(frame_h, th, ny, j), tw, th};
    *count = (int) n;
    return 0;
}

// ---- tensors ----
int snnb_tensor_alloc(snnb_context* ctx, int n, int h, int w, int c, snnb_tensor** out) { return tensor_alloc(ctx, n, h, w, c, out); }
int snnb_tensor_free(snnb_tensor* t) {
    if (!t) return 0;
    if (t->owns && t->hi) cudaFree(t->hi);
    if (t->feed_hi) cudaFree(t->feed_hi);
    delete t;
    return 0;
}
int snnb_debug_feed_plan(int k, int stride, int pad_x, int ic, int out[5]) {
    FeedPlan fp;
    if (!out || !make_feed_plan(k, stride, pad_x, ic, fp)) return 0;
    out[0] = fp.px, out[1] = fp.d, out[2] = fp.nch, out[3] = fp.ksteps, out[4] = fp.rows_per_panel;
    return 1;
}
int snnb_debug_conv_launch(const int query[24], int out[59]) {
    SNNB_REQUIRE(query && out, "snnb_debug_conv_launch: null argument");
    ConvQuery q;
    q.in_h = query[0], q.in_w = query[1], q.in_c = query[2], q.out_h = query[3], q.out_w = query[4], q.out_c = query[5];
    q.k = query[6], q.stride = query[7], q.pad_x = query[8], q.pad_y = query[9], q.pad_mode = query[10];
    q.residual = query[11] != 0, q.algo = query[12], q.may_prepad = query[13] != 0, q.may_feed = query[14] != 0;
    q.row_stride = query[15], q.row_pad = query[16], q.feed_pad = query[17];
    q.n = query[18], q.precision = query[19], q.in_lo = query[20] != 0, q.out_lo = query[21] != 0, q.stream_k = query[22] != 0, q.sm_count = query[23];
    SNNB_REQUIRE(q.n > 0 && q.sm_count > 0, "snnb_debug_conv_launch: batch %d and SM count %d must be positive", q.n, q.sm_count);
    const ConvPlan p = plan_conv(q);
    const RowPlan rp = p.path == CONV_ROWWIN || p.path == CONV_ROWWIN_FEED ? p.rp : RowPlan();
    const int v[43] = {p.path, p.pad_x, p.pad_y, p.pad_mode, p.prepad_h, p.prepad_w, p.feed_h, p.feed_w, p.feed_py, p.feed_px,
                       p.n, p.terms, p.n_blk, p.tiles_x, p.grid,
                       p.tw, p.th, p.tn, p.tiles_y, p.tiles_n, p.tiles_oc, p.ksplit, p.kb_per_split, p.sk, p.sk_dp, p.sk_ctas, (int) p.sk_units,
                       p.partial_tiles, p.partial_slots,
                       p.fks, p.panels, p.rows_per_stage, p.wrows, p.stages, (int) p.row_bytes, (int) p.lo_off, (int) p.stage_bytes, (int) p.b_bytes,
                       (int) p.feed_seg_bytes, rp.parities, rp.ksteps, rp.dmin[0], rp.dmin[1]};
    std::copy(v, v + 43, out);
    std::copy(rp.ks_parity, rp.ks_parity + 8, out + 43);
    std::copy(rp.ks_erel, rp.ks_erel + 8, out + 51);
    return 0;
}
int snnb_debug_conv_plan(const int query[18], int out[10]) {
    SNNB_REQUIRE(query && out, "snnb_debug_conv_plan: null argument");
    // the path, pads and copies do not depend on the batch, product form or SM count
    int q[24], full[59];
    const int launch[6] = {1, SNNB_PRECISION_FP32X3, 1, 1, 0, 1};
    std::copy(query, query + 18, q);
    std::copy(launch, launch + 6, q + 18);
    if (int rc = snnb_debug_conv_launch(q, full)) return rc;
    std::copy(full, full + 10, out);
    return 0;
}
int snnb_debug_streamk_schedule(int tiles, int num_kb, int sms, int* rows, int capacity) {
    SNNB_REQUIRE(rows || capacity == 0, "snnb_debug_streamk_schedule: null buffer");
    return streamk_schedule(tiles, num_kb, sms, rows, capacity);
}
int snnb_debug_count_body(const int* sizes, int num_sizes, int batch, int count) {
    if (!(sizes || num_sizes == 0) || num_sizes < 0 || batch < 1) {
        set_error("snnb_debug_count_body: %d sizes at %p, batch %d", num_sizes, (const void*) sizes, batch);
        return -1; // every size is >= 0
    }
    return count_body(sizes, num_sizes, batch, count);
}
int snnb_debug_last_conv_variant(snnb_context* ctx, int out[6]) {
    SNNB_REQUIRE(ctx && out, "snnb_debug_last_conv_variant: null argument");
    for (int i = 0; i < 6; ++i) out[i] = ctx->last_conv[i];
    return 0;
}
int snnb_debug_launches(snnb_context* ctx, char* buf, int cap, int clear) {
    if (!ctx || !buf || cap < 1) {
        set_error("snnb_debug_launches: context %p, buffer %p of %d bytes", (void*) ctx, (void*) buf, cap);
        return -1;
    }
    const std::string& log = ctx->launch_log;
    const size_t n         = std::min(log.size(), (size_t) cap - 1);
    std::copy(log.data(), log.data() + n, buf);
    buf[n] = '\0';
    const int len = (int) log.size();
    if (clear) ctx->launch_log.clear();
    return len;
}
int snnb_tensor_planes(const snnb_tensor* t, void** hi, void** lo, int* cp) {
    SNNB_REQUIRE(t && hi && lo && cp, "snnb_tensor_planes: null argument");
    *hi = t->hi, *lo = t->lo, *cp = t->cp;
    return 0;
}
int snnb_tensor_dims(const snnb_tensor* t, int* n, int* h, int* w, int* c) {
    SNNB_REQUIRE(t, "snnb_tensor_dims: null tensor");
    if (n) *n = t->n;
    if (h) *h = t->h;
    if (w) *w = t->w;
    if (c) *c = t->c;
    return 0;
}
int snnb_tensor_upload_nhwc(snnb_context* ctx, snnb_tensor* t, const float* host) {
    SNNB_REQUIRE(ctx && t && host, "snnb_tensor_upload_nhwc: null argument");
    const size_t bytes = t->pixels() * t->c * sizeof(float);
    if (ensure_stage(ctx, bytes)) return 1;
    SNNB_CUDA_OK(cudaMemcpyAsync(ctx->stage_dev, host, bytes, cudaMemcpyHostToDevice, ctx->stream));
    if (launch_split_f32(ctx, ctx->stage_dev, t)) return 1;
    SNNB_CUDA_OK(cudaStreamSynchronize(ctx->stream));
    return 0;
}
int snnb_tensor_download_nhwc(snnb_context* ctx, const snnb_tensor* t, float* host) {
    SNNB_REQUIRE(ctx && t && host, "snnb_tensor_download_nhwc: null argument");
    const size_t bytes = t->pixels() * t->c * sizeof(float);
    if (ensure_stage(ctx, bytes)) return 1;
    if (launch_merge_f32(ctx, t, ctx->stage_dev)) return 1;
    SNNB_CUDA_OK(cudaMemcpyAsync(host, ctx->stage_dev, bytes, cudaMemcpyDeviceToHost, ctx->stream));
    SNNB_CUDA_OK(cudaStreamSynchronize(ctx->stream));
    return 0;
}

// C4HW4 <-> NHWC on the host (API-edge convenience for callers holding reference-layout textures).
static void c4_to_nhwc(const float* c4, int N, int H, int W, int C, float* nhwc) {
    const int D = (C + 3) / 4;
    for (int n = 0; n < N; ++n)
        for (int y = 0; y < H; ++y)
            for (int x = 0; x < W; ++x)
                for (int c = 0; c < C; ++c)
                    nhwc[(((size_t) n * H + y) * W + x) * C + c] = c4[((((size_t) n * D + c / 4) * H + y) * W + x) * 4 + (c % 4)];
}
static void nhwc_to_c4(const float* nhwc, int N, int H, int W, int C, float* c4) {
    const int D = (C + 3) / 4;
    memset(c4, 0, sizeof(float) * (size_t) N * D * H * W * 4);
    for (int n = 0; n < N; ++n)
        for (int y = 0; y < H; ++y)
            for (int x = 0; x < W; ++x)
                for (int c = 0; c < C; ++c)
                    c4[((((size_t) n * D + c / 4) * H + y) * W + x) * 4 + (c % 4)] = nhwc[(((size_t) n * H + y) * W + x) * C + c];
}
int snnb_tensor_upload_c4hw4(snnb_context* ctx, snnb_tensor* t, const float* host_c4) {
    SNNB_REQUIRE(ctx && t && host_c4, "snnb_tensor_upload_c4hw4: null argument");
    std::vector<float> tmp(t->pixels() * t->c);
    c4_to_nhwc(host_c4, t->n, t->h, t->w, t->c, tmp.data());
    return snnb_tensor_upload_nhwc(ctx, t, tmp.data());
}
int snnb_tensor_download_c4hw4(snnb_context* ctx, const snnb_tensor* t, float* host_c4) {
    SNNB_REQUIRE(ctx && t && host_c4, "snnb_tensor_download_c4hw4: null argument");
    std::vector<float> tmp(t->pixels() * t->c);
    if (snnb_tensor_download_nhwc(ctx, t, tmp.data())) return 1;
    nhwc_to_c4(tmp.data(), t->n, t->h, t->w, t->c, host_c4);
    return 0;
}
int snnb_tensor_dump(snnb_context* ctx, const snnb_tensor* t, const char* path) {
    SNNB_REQUIRE(ctx && t && path, "snnb_tensor_dump: null argument");
    const int D = (t->c + 3) / 4;
    std::vector<float> c4((size_t) t->n * D * t->h * t->w * 4);
    if (snnb_tensor_download_c4hw4(ctx, t, c4.data())) return 1;
    for (int n = 0; n < t->n; ++n) {
        std::string p = path;
        if (t->n > 1) p += ".n" + std::to_string(n);
        FILE* f = fopen(p.c_str(), "wb");
        SNNB_REQUIRE(f, "snnb_tensor_dump: cannot open %s", p.c_str());
        char header[32];
        memset(header, 0, sizeof(header));
        snprintf(header, sizeof(header), "%d %d %d %d", t->w, t->h, D, t->c); // image.cpp:216-245: "W H D C"
        fwrite(header, 1, sizeof(header), f);
        fwrite(c4.data() + (size_t) n * D * t->h * t->w * 4, sizeof(float), (size_t) D * t->h * t->w * 4, f);
        fclose(f);
    }
    return 0;
}

// ---- weights ----
static int make_weights(snnb_context* ctx, const PackedHost& p, snnb_weights** out) {
    auto w       = std::make_unique<snnb_weights>();
    size_t bytes = p.device_bytes();
    SNNB_CUDA_OK(cudaMalloc(&w->owned, bytes ? bytes : 256));
    if (place_weights(ctx, p, (char*) w->owned, w.get())) {
        cudaFree(w->owned);
        return 1;
    }
    *out = w.release();
    return 0;
}
int snnb_weights_pack_conv2d(snnb_context* ctx, const snnb_conv_desc* d, const float* w_oihw, const float* bias, const float* g, const float* b,
                             const float* m, const float* v, snnb_weights** out) {
    SNNB_REQUIRE(ctx && d && w_oihw && out, "snnb_weights_pack_conv2d: null argument");
    SNNB_REQUIRE(d->in_channels > 0 && d->out_channels > 0 && d->kernel > 0, "snnb_weights_pack_conv2d: bad desc");
    PackedHost p;
    pack_conv2d_host(d->in_channels, d->out_channels, d->kernel, w_oihw, bias, g, b, m, v, p);
    pack_rowwin_host(p, d->stride, d->pad_x);
    return make_weights(ctx, p, out);
}
int snnb_weights_pack_depthwise(snnb_context* ctx, const snnb_conv_desc* d, const float* w_chw, const float* bias, const float* g, const float* b,
                                const float* m, const float* v, snnb_weights** out) {
    SNNB_REQUIRE(ctx && d && w_chw && out, "snnb_weights_pack_depthwise: null argument");
    SNNB_REQUIRE(d->in_channels > 0 && d->in_channels == d->out_channels, "snnb_weights_pack_depthwise: depth multiplier != 1 is not supported "
                                                                           "(as in the reference, modelparser.cpp:821)");
    PackedHost p;
    pack_depthwise_host(d->in_channels, d->kernel, w_chw, bias, g, b, m, v, p);
    return make_weights(ctx, p, out);
}
int snnb_weights_pack_dense(snnb_context* ctx, int n_in, int n_out, const float* kernel, const float* bias, snnb_weights** out) {
    SNNB_REQUIRE(ctx && kernel && out && n_in > 0 && n_out > 0, "snnb_weights_pack_dense: bad argument");
    PackedHost p; // [out][in] row-major == OIHW with k = 1
    pack_conv2d_host(n_in, n_out, 1, kernel, bias, nullptr, nullptr, nullptr, nullptr, p);
    p.kind = 3;
    return make_weights(ctx, p, out);
}
int snnb_weights_pack_channels(snnb_context* ctx, int channels, const float* g, const float* b, const float* m, const float* v, snnb_weights** out) {
    SNNB_REQUIRE(ctx && out && channels > 0, "snnb_weights_pack_channels: bad argument");
    PackedHost p;
    pack_channels_host(channels, g, b, m, v, p);
    return make_weights(ctx, p, out);
}
int snnb_weights_free(snnb_weights* w) {
    if (!w) return 0;
    if (w->owned) cudaFree(w->owned);
    delete w;
    return 0;
}

// ---- operators ----
int snnb_conv2d_launch(snnb_context* ctx, const snnb_conv_desc* d, const snnb_weights* w, const snnb_tensor* in, const snnb_tensor* residual,
                       snnb_tensor* out) {
    SNNB_REQUIRE(ctx && d && w && in && out, "snnb_conv2d_launch: null argument");
    SNNB_REQUIRE(w->kind == 1 || w->kind == 3, "snnb_conv2d_launch: weights were not packed for conv2d");
    SNNB_REQUIRE(in->c == w->in_ch && out->c == w->out_ch && d->kernel == w->kernel, "snnb_conv2d_launch: tensor channels (%d -> %d, k%d) do not match the weights (%d -> %d, k%d)",
                 in->c, out->c, d->kernel, w->in_ch, w->out_ch, w->kernel);
    SNNB_REQUIRE(in->n == out->n, "snnb_conv2d_launch: batch mismatch");
    if (residual) CHECK_DIMS_EQ(residual, out, "snnb_conv2d_launch(residual)");
    ConvQuery q;
    q.in_h = in->h, q.in_w = in->w, q.in_c = in->c, q.out_h = out->h, q.out_w = out->w, q.out_c = out->c;
    q.k = d->kernel, q.stride = d->stride, q.pad_x = d->pad_x, q.pad_y = d->pad_y, q.pad_mode = d->pad_mode;
    q.residual = residual != nullptr, q.algo = d->algo;
    q.row_stride = w->row_stride, q.row_pad = w->row_pad, q.feed_pad = w->feed_pad;
    q.n = out->n, q.precision = ctx->precision, q.in_lo = in->lo != nullptr, q.out_lo = out->lo != nullptr, q.sm_count = ctx->sm_count;
    q.stream_k = d->algo == SNNB_ALGO_TCGEN05_STREAMK;
    ConvArgs a {in, residual, out, w, d->kernel, d->stride, d->pad_x, d->pad_y, d->pad_mode, d->activation, d->leaky_alpha};
    return launch_conv2d(ctx, a, plan_conv(q));
}
int snnb_depthwise_launch(snnb_context* ctx, const snnb_conv_desc* d, const snnb_weights* w, const snnb_tensor* in, snnb_tensor* out) {
    SNNB_REQUIRE(ctx && d && w && in && out, "snnb_depthwise_launch: null argument");
    SNNB_REQUIRE(w->kind == 2 && in->c == w->in_ch && out->c == in->c && d->kernel == w->kernel, "snnb_depthwise_launch: weights/tensor mismatch");
    SNNB_REQUIRE(in->n == out->n, "snnb_depthwise_launch: batch mismatch");
    // the depthwise kernels clip the window to the input, which is zero padding; replicate or reflect would silently read zeros
    SNNB_REQUIRE(d->pad_mode == SNNB_PAD_NONE || d->pad_mode == SNNB_PAD_CONSTANT, "snnb_depthwise_launch: pad_mode %d; depthwise pads with zeros only (NONE or CONSTANT)",
                 d->pad_mode);
    ConvArgs a {in, nullptr, out, w, d->kernel, d->stride, d->pad_x, d->pad_y, SNNB_PAD_CONSTANT, d->activation, d->leaky_alpha};
    return launch_depthwise(ctx, a);
}
int snnb_maxpool_launch(snnb_context* ctx, int kernel, int stride, const snnb_tensor* in, snnb_tensor* out) {
    SNNB_REQUIRE(ctx && in && out && kernel > 0 && stride > 0 && in->c == out->c && in->n == out->n, "snnb_maxpool_launch: bad argument");
    // every window must START inside the input (pool windows are clipped at the bottom/right edge, never padded top/left)
    SNNB_REQUIRE((long long) (out->w - 1) * stride < in->w && (long long) (out->h - 1) * stride < in->h, "snnb_maxpool_launch: output %dx%d does not fit input %dx%d at stride %d", out->h, out->w, in->h, in->w, stride);
    return launch_pool(ctx, in, out, kernel, stride, false);
}
int snnb_avgpool_launch(snnb_context* ctx, int kernel, int stride, const snnb_tensor* in, snnb_tensor* out) {
    SNNB_REQUIRE(ctx && in && out && kernel > 0 && stride > 0 && in->c == out->c && in->n == out->n, "snnb_avgpool_launch: bad argument");
    // every window must START inside the input (pool windows are clipped at the bottom/right edge, never padded top/left)
    SNNB_REQUIRE((long long) (out->w - 1) * stride < in->w && (long long) (out->h - 1) * stride < in->h, "snnb_avgpool_launch: output %dx%d does not fit input %dx%d at stride %d", out->h, out->w, in->h, in->w, stride);
    return launch_pool(ctx, in, out, kernel, stride, true);
}
int snnb_add_launch(snnb_context* ctx, int act, float alpha, const snnb_tensor* a, const snnb_tensor* b, snnb_tensor* out) {
    SNNB_REQUIRE(ctx && a && b && out, "snnb_add_launch: null argument");
    CHECK_DIMS_EQ(a, b, "snnb_add_launch");
    CHECK_DIMS_EQ(a, out, "snnb_add_launch");
    return launch_add(ctx, a, b, out, act, alpha);
}
int snnb_batchnorm_launch(snnb_context* ctx, const snnb_weights* w, int act, float alpha, const snnb_tensor* in, snnb_tensor* out) {
    SNNB_REQUIRE(ctx && w && in && out && w->kind == 4 && w->in_ch == in->c, "snnb_batchnorm_launch: bad argument");
    CHECK_DIMS_EQ(in, out, "snnb_batchnorm_launch");
    return launch_batchnorm(ctx, in, out, w, act, alpha);
}
int snnb_activation_launch(snnb_context* ctx, int act, float alpha, const snnb_tensor* in, snnb_tensor* out) {
    SNNB_REQUIRE(ctx && in && out, "snnb_activation_launch: null argument");
    CHECK_DIMS_EQ(in, out, "snnb_activation_launch");
    return launch_activation(ctx, in, out, act, alpha);
}
int snnb_softmax_launch(snnb_context* ctx, const snnb_tensor* in, snnb_tensor* out) {
    SNNB_REQUIRE(ctx && in && out, "snnb_softmax_launch: null argument");
    CHECK_DIMS_EQ(in, out, "snnb_softmax_launch");
    return launch_softmax(ctx, in, out);
}
int snnb_flatten_launch(snnb_context* ctx, const snnb_tensor* in, snnb_tensor* out) {
    SNNB_REQUIRE(ctx && in && out && out->n == in->n && out->h == 1 && out->w == 1 && out->c == in->h * in->w * in->c, "snnb_flatten_launch: bad dims");
    return launch_flatten(ctx, in, out);
}
int snnb_dense_launch(snnb_context* ctx, const snnb_weights* w, int act, float alpha, const snnb_tensor* in, snnb_tensor* out) {
    SNNB_REQUIRE(ctx && w && in && out && (w->kind == 3 || w->kind == 1), "snnb_dense_launch: bad argument");
    SNNB_REQUIRE(in->h * in->w * in->c == w->in_ch && out->c == w->out_ch && out->h == 1 && out->w == 1 && in->n == out->n,
                 "snnb_dense_launch: dims do not match the weights (%d -> %d)", w->in_ch, w->out_ch);
    snnb_tensor* flat = nullptr;
    if (in->h * in->w != 1 && tensor_alloc(ctx, in->n, 1, 1, w->in_ch, &flat)) return 1;
    const snnb_tensor* x = flat ? flat : in;
    ConvQuery q          = dense_query(out->n, x->c, out->c, ctx->precision, x->lo && out->lo, ctx->sm_count);
    q.row_stride = w->row_stride, q.row_pad = w->row_pad, q.feed_pad = w->feed_pad;
    const int rc = launch_dense(ctx, in, flat, out, w, act, alpha, plan_conv(q));
    if (flat) {
        cudaStreamSynchronize(ctx->stream);
        snnb_tensor_free(flat);
    }
    return rc;
}
int snnb_argmax1(snnb_context* ctx, const snnb_tensor* in, int* host_idx) {
    SNNB_REQUIRE(ctx && in && host_idx, "snnb_argmax1: null argument");
    // argmax_kernel scans the channels of pixel 0 of each image
    SNNB_REQUIRE(in->h == 1 && in->w == 1, "snnb_argmax1: input is %dx%d per image; it must be [N,1,1,C]", in->h, in->w);
    if (ensure_stage(ctx, sizeof(int) * in->n)) return 1;
    int* dev = reinterpret_cast<int*>(ctx->stage_dev);
    if (launch_argmax(ctx, in, dev)) return 1;
    SNNB_CUDA_OK(cudaMemcpyAsync(host_idx, dev, sizeof(int) * in->n, cudaMemcpyDeviceToHost, ctx->stream));
    SNNB_CUDA_OK(cudaStreamSynchronize(ctx->stream));
    for (int i = 0; i < in->n; ++i) host_idx[i] += 1; // core.cpp:228-233: 1-based
    return 0;
}
int snnb_concat_launch(snnb_context* ctx, const snnb_tensor* a, const snnb_tensor* b, snnb_tensor* out) {
    SNNB_REQUIRE(ctx && a && b && out, "snnb_concat_launch: null argument");
    SNNB_REQUIRE(a->n == b->n && a->h == b->h && a->w == b->w && out->n == a->n && out->h == a->h && out->w == a->w && out->c == a->c + b->c,
                 "snnb_concat_launch: bad dims");
    return launch_concat(ctx, a, b, out);
}
int snnb_upsample_launch(snnb_context* ctx, float scale, int bilinear, const snnb_tensor* in, snnb_tensor* out) {
    SNNB_REQUIRE(ctx && in && out && scale > 0 && in->c == out->c && in->n == out->n, "snnb_upsample_launch: bad argument");
    return launch_upsample(ctx, in, out, scale, bilinear != 0);
}
int snnb_pad_launch(snnb_context* ctx, int pad_x, int pad_y, int mode, const snnb_tensor* in, snnb_tensor* out) {
    SNNB_REQUIRE(ctx && in && out && in->c == out->c && in->n == out->n, "snnb_pad_launch: bad argument");
    return launch_pad(ctx, in, out, pad_x, pad_y, mode);
}
int snnb_instancenorm_launch(snnb_context* ctx, const snnb_weights* w, int act, float alpha, const snnb_tensor* in, snnb_tensor* out) {
    SNNB_REQUIRE(ctx && w && in && out && w->kind == 4 && w->in_ch == in->c, "snnb_instancenorm_launch: bad argument");
    CHECK_DIMS_EQ(in, out, "snnb_instancenorm_launch");
    return launch_instancenorm(ctx, in, out, w, act, alpha);
}
int snnb_subpixel_launch(snnb_context* ctx, int r, const snnb_tensor* in, snnb_tensor* out) {
    SNNB_REQUIRE(ctx && in && out && r > 0 && in->c == r * r && out->c == 1 && out->h == in->h * r && out->w == in->w * r && in->n == out->n,
                 "snnb_subpixel_launch: bad dims");
    return launch_subpixel(ctx, in, out, r);
}

// ---- timers ----
int snnb_timer_create(snnb_context* ctx, snnb_timer** out) {
    SNNB_REQUIRE(ctx && out, "snnb_timer_create: null argument");
    auto t = std::make_unique<snnb_timer>();
    t->ctx = ctx;
    SNNB_CUDA_OK(cudaEventCreate(&t->e0));
    SNNB_CUDA_OK(cudaEventCreate(&t->e1));
    *out = t.release();
    return 0;
}
int snnb_timer_start(snnb_timer* t) {
    SNNB_REQUIRE(t, "snnb_timer_start: null timer");
    SNNB_CUDA_OK(cudaEventRecord(t->e0, t->ctx->stream));
    return 0;
}
int snnb_timer_stop(snnb_timer* t) {
    SNNB_REQUIRE(t, "snnb_timer_stop: null timer");
    SNNB_CUDA_OK(cudaEventRecord(t->e1, t->ctx->stream));
    return 0;
}
int snnb_timer_elapsed_ms(snnb_timer* t, float* ms) {
    SNNB_REQUIRE(t && ms, "snnb_timer_elapsed_ms: null argument");
    SNNB_CUDA_OK(cudaEventSynchronize(t->e1));
    SNNB_CUDA_OK(cudaEventElapsedTime(ms, t->e0, t->e1));
    return 0;
}
int snnb_timer_destroy(snnb_timer* t) {
    if (!t) return 0;
    cudaEventDestroy(t->e0);
    cudaEventDestroy(t->e1);
    delete t;
    return 0;
}

// ---- launch capture -----------------------------------------------------------------------------------------
int snnb_graph_capture_begin(snnb_context* ctx) {
    SNNB_REQUIRE(ctx, "snnb_graph_capture_begin: null context");
    SNNB_CUDA_OK(cudaSetDevice(ctx->device));
    cudaStreamCaptureStatus st = cudaStreamCaptureStatusNone;
    SNNB_CUDA_OK(cudaStreamIsCapturing(ctx->stream, &st));
    SNNB_REQUIRE(st == cudaStreamCaptureStatusNone, "snnb_graph_capture_begin: the context is already capturing");
    SNNB_CUDA_OK(cudaStreamBeginCapture(ctx->stream, cudaStreamCaptureModeThreadLocal));
    return 0;
}
int snnb_graph_capture_end(snnb_context* ctx, snnb_graph** out) {
    SNNB_REQUIRE(ctx && out, "snnb_graph_capture_end: null argument");
    cudaGraph_t g = nullptr;
    const cudaError_t e = cudaStreamEndCapture(ctx->stream, &g);
    if (e != cudaSuccess || !g) {
        cudaGetLastError();
        set_error("snnb_graph_capture_end: capture failed (%s); a launch inside the region reported an error or allocated memory", cudaGetErrorString(e));
        return 1;
    }
    cudaGraphExec_t ex = nullptr;
    const cudaError_t e2 = cudaGraphInstantiate(&ex, g, 0);
    if (e2 != cudaSuccess) {
        cudaGraphDestroy(g);
        set_error("snnb_graph_capture_end: cudaGraphInstantiate failed (%s)", cudaGetErrorString(e2));
        return 1;
    }
    auto* h = new snnb_graph();
    h->ctx = ctx, h->graph = g, h->exec = ex;
    *out = h;
    return 0;
}
int snnb_graph_launch(snnb_graph* g) {
    SNNB_REQUIRE(g && g->exec, "snnb_graph_launch: null graph");
    SNNB_CUDA_OK(cudaSetDevice(g->ctx->device));
    SNNB_CUDA_OK(cudaGraphLaunch(g->exec, g->ctx->stream));
    return 0;
}
int snnb_graph_destroy(snnb_graph* g) {
    if (!g) return 0;
    if (g->exec) cudaGraphExecDestroy(g->exec);
    if (g->graph) cudaGraphDestroy(g->graph);
    delete g;
    return 0;
}

} // extern "C"
