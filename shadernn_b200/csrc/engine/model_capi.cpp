// extern "C" surface for the whole-model engine (snnb_model_*). See include/snnb.h.
#include <dlfcn.h>

#include <cstring>

#include "engine.h"

using namespace snnb;

struct snnb_model {
    std::unique_ptr<snn::MixedInferenceCore> core;
};

static void copyStr(char* dst, int cap, const std::string& s) {
    if (!dst || cap <= 0) return;
    strncpy(dst, s.c_str(), (size_t) cap - 1);
    dst[cap - 1] = 0;
}

extern "C" {

int snnb_model_load_json(snnb_context* ctx, const char* json_path, const snnb_model_options* opt, snnb_model** out) {
    SNNB_REQUIRE(ctx && json_path && out, "snnb_model_load_json: null argument");
    snn::dp::ShaderGenOptions o;
    if (opt) {
        o.batch              = opt->batch > 0 ? (uint32_t) opt->batch : 1;
        o.desiredInputWidth  = opt->input_width > 0 ? (uint32_t) opt->input_width : 0;
        o.desiredInputHeight = opt->input_height > 0 ? (uint32_t) opt->input_height : 0;
        o.convAlgo           = opt->conv_algo;
        o.useCudaGraph       = opt->use_cuda_graph != 0;
        o.fuse               = opt->fuse != 0;
        o.precision          = opt->precision;
        SNNB_REQUIRE(o.precision >= SNNB_PRECISION_FP32X3 && o.precision <= SNNB_PRECISION_FP16, "snnb_model_load_json: unknown precision %d", o.precision);
    }
    SNNB_CUDA_OK(cudaSetDevice(ctx->device));
    std::string err;
    std::unique_ptr<snn::MixedInferenceCore> core;
    try {
        core = snn::MixedInferenceCore::create(ctx, json_path, o, err);
    } catch (std::exception& e) { err = e.what(); }
    if (!core) {
        set_error("snnb_model_load_json(%s): %s", json_path, err.c_str());
        return 1;
    }
    auto* m = new snnb_model();
    m->core = std::move(core);
    *out    = m;
    return 0;
}

int snnb_model_destroy(snnb_model* m) {
    if (m && m->core && m->core->ctx) cudaSetDevice(m->core->ctx->device);
    delete m;
    return 0;
}

int snnb_model_num_layers(const snnb_model* m) { return m ? (int) m->core->layers.size() : -1; }

int snnb_model_layer_info(const snnb_model* m, int i, char* name, int name_cap, char* type, int type_cap, int* n, int* h, int* w, int* c) {
    SNNB_REQUIRE(m && i >= 0 && i < (int) m->core->layers.size(), "snnb_model_layer_info: bad index");
    auto* L = m->core->layers[i].get();
    copyStr(name, name_cap, L->name);
    copyStr(type, type_cap, L->typeName);
    // dims from the graph (valid for fused-away layers too)
    for (size_t k = 0; k < m->core->graph.sorted.size(); ++k)
        if (m->core->graph.sorted[k] == L) {
            const auto& d = m->core->graph.outputDims[k];
            if (n) *n = m->core->batch();
            if (h) *h = (int) d.height;
            if (w) *w = (int) d.width;
            if (c) *c = (int) d.depth;
        }
    return 0;
}

int snnb_model_num_inputs(const snnb_model* m) { return m ? (int) m->core->inputLayers.size() : -1; }
int snnb_model_num_outputs(const snnb_model* m) { return m ? (int) m->core->outputLayers.size() : -1; }

static int dimsOf(const snnb_tensor* t, int* n, int* h, int* w, int* c) {
    SNNB_REQUIRE(t, "tensor not materialised");
    return snnb_tensor_dims(t, n, h, w, c);
}
int snnb_model_input_dims(const snnb_model* m, int idx, int* n, int* h, int* w, int* c) {
    SNNB_REQUIRE(m && idx >= 0 && idx < (int) m->core->inputLayers.size(), "snnb_model_input_dims: bad index");
    return dimsOf(m->core->inputLayers[idx]->output, n, h, w, c);
}
int snnb_model_output_dims(const snnb_model* m, int idx, int* n, int* h, int* w, int* c) {
    SNNB_REQUIRE(m && idx >= 0 && idx < (int) m->core->outputLayers.size(), "snnb_model_output_dims: bad index");
    auto* L = m->core->outputLayers[idx];
    if (L->typeName == "YOLO") {
        if (n) *n = m->core->batch();
        if (h) *h = 100;
        if (w) *w = 6;
        if (c) *c = 1;
        return 0;
    }
    return dimsOf(L->output, n, h, w, c);
}

int snnb_model_run(snnb_model* m, const float* host_input, float* host_output, size_t out_capacity, int* classes) {
    SNNB_REQUIRE(m && host_input, "snnb_model_run: null argument");
    SNNB_CUDA_OK(cudaSetDevice(m->core->ctx->device));
    return m->core->run(host_input, host_output, out_capacity, classes);
}
int snnb_model_submit(snnb_model* m, const float* host_input, float* host_output, size_t out_capacity, int* classes, int* ticket) {
    SNNB_REQUIRE(m, "snnb_model_submit: null model");
    SNNB_CUDA_OK(cudaSetDevice(m->core->ctx->device));
    return m->core->submit(host_input, host_output, out_capacity, classes, ticket);
}
int snnb_model_submit_u8(snnb_model* m, const uint8_t* host_input_u8, const float* mean4, const float* norm4, float* host_output, size_t out_capacity, int* classes,
                         int* ticket) {
    SNNB_REQUIRE(m, "snnb_model_submit_u8: null model");
    SNNB_CUDA_OK(cudaSetDevice(m->core->ctx->device));
    return m->core->submitU8(host_input_u8, mean4, norm4, host_output, out_capacity, classes, ticket);
}
int snnb_model_submit_image(snnb_model* m, const snnb_image_io* io, int* ticket) {
    SNNB_REQUIRE(m && io && ticket, "snnb_model_submit_image: null argument");
    SNNB_CUDA_OK(cudaSetDevice(m->core->ctx->device));
    return m->core->submitImage(*io, ticket);
}
int snnb_model_wait(snnb_model* m, int ticket) {
    SNNB_REQUIRE(m, "snnb_model_wait: null model");
    SNNB_CUDA_OK(cudaSetDevice(m->core->ctx->device));
    return m->core->wait(ticket);
}
int snnb_model_run_device(snnb_model* m, const snnb_device_buffer* inputs, int num_inputs, const snnb_device_buffer* outputs, int num_outputs,
                          int* classes_1based_dev, void* stream) {
    SNNB_REQUIRE(m, "snnb_model_run_device: null model");
    SNNB_CUDA_OK(cudaSetDevice(m->core->ctx->device));
    return m->core->runDevice(inputs, num_inputs, outputs, num_outputs, classes_1based_dev, static_cast<cudaStream_t>(stream));
}
int snnb_model_detect_device(snnb_model* m, const snnb_device_buffer* inputs, int num_inputs, float* rows_dev, int max_rows, int* counts_dev, void* stream) {
    SNNB_REQUIRE(m, "snnb_model_detect_device: null model");
    SNNB_CUDA_OK(cudaSetDevice(m->core->ctx->device));
    return m->core->detectDevice(inputs, num_inputs, rows_dev, max_rows, counts_dev, static_cast<cudaStream_t>(stream));
}
int snnb_model_run_frames(snnb_model* m, const snnb_frames* frames, const snnb_device_buffer* outputs, int num_outputs, int* classes_1based_dev, void* stream) {
    SNNB_REQUIRE(m, "snnb_model_run_frames: null model");
    SNNB_CUDA_OK(cudaSetDevice(m->core->ctx->device));
    return m->core->runFrames(frames, outputs, num_outputs, classes_1based_dev, static_cast<cudaStream_t>(stream));
}
int snnb_model_detect_frames(snnb_model* m, const snnb_frames* frames, float* rows_dev, int max_rows, int* counts_dev, void* stream) {
    SNNB_REQUIRE(m, "snnb_model_detect_frames: null model");
    SNNB_CUDA_OK(cudaSetDevice(m->core->ctx->device));
    return m->core->detectFrames(frames, rows_dev, max_rows, counts_dev, static_cast<cudaStream_t>(stream));
}
int snnb_model_transform_frames(snnb_model* m, const snnb_frames* frames, const snnb_frames_out* out, void* stream) {
    SNNB_REQUIRE(m, "snnb_model_transform_frames: null model");
    SNNB_CUDA_OK(cudaSetDevice(m->core->ctx->device));
    return m->core->transformFrames(frames, out, static_cast<cudaStream_t>(stream));
}
int snnb_model_transform_luma(snnb_model* m, const snnb_frames* frames, const snnb_frames_out* out, void* stream) {
    SNNB_REQUIRE(m, "snnb_model_transform_luma: null model");
    SNNB_CUDA_OK(cudaSetDevice(m->core->ctx->device));
    return m->core->transformLuma(frames, out, static_cast<cudaStream_t>(stream));
}
int snnb_model_segment_frames(snnb_model* m, const snnb_frames* frames, int luma, const snnb_labels_out* out, void* stream) {
    SNNB_REQUIRE(m, "snnb_model_segment_frames: null model");
    SNNB_CUDA_OK(cudaSetDevice(m->core->ctx->device));
    return m->core->segmentFrames(frames, luma != 0, out, static_cast<cudaStream_t>(stream));
}
int snnb_model_run_rois(snnb_model* m, const snnb_frames* frames, int num_frames, const snnb_roi* rois_dev, const int* count_dev,
                        const snnb_device_buffer* outputs, int num_outputs, int* classes_1based_dev, void* stream) {
    SNNB_REQUIRE(m, "snnb_model_run_rois: null model");
    SNNB_CUDA_OK(cudaSetDevice(m->core->ctx->device));
    return m->core->runRois(frames, num_frames, rois_dev, count_dev, outputs, num_outputs, classes_1based_dev, static_cast<cudaStream_t>(stream));
}
int snnb_model_run_frame_list(snnb_model* m, const snnb_frame_list* frames, const snnb_device_buffer* outputs, int num_outputs, int* classes_1based_dev,
                              void* stream) {
    SNNB_REQUIRE(m, "snnb_model_run_frame_list: null model");
    SNNB_CUDA_OK(cudaSetDevice(m->core->ctx->device));
    return m->core->runFrameList(frames, outputs, num_outputs, classes_1based_dev, static_cast<cudaStream_t>(stream));
}
int snnb_model_detect_frame_list(snnb_model* m, const snnb_frame_list* frames, float* rows_dev, int max_rows, int* counts_dev, void* stream) {
    SNNB_REQUIRE(m, "snnb_model_detect_frame_list: null model");
    SNNB_CUDA_OK(cudaSetDevice(m->core->ctx->device));
    return m->core->detectFrameList(frames, rows_dev, max_rows, counts_dev, static_cast<cudaStream_t>(stream));
}
int snnb_model_run_rois_list(snnb_model* m, const snnb_frame_list* frames, const snnb_roi* rois_dev, const int* count_dev, const snnb_device_buffer* outputs,
                             int num_outputs, int* classes_1based_dev, void* stream) {
    SNNB_REQUIRE(m, "snnb_model_run_rois_list: null model");
    SNNB_CUDA_OK(cudaSetDevice(m->core->ctx->device));
    return m->core->runRoisList(frames, rois_dev, count_dev, outputs, num_outputs, classes_1based_dev, static_cast<cudaStream_t>(stream));
}
int snnb_model_detect_rois(snnb_model* m, const snnb_frames* frames, int num_frames, const snnb_roi* rois_dev, const int* count_dev, float* rows_dev,
                           int max_rows, int* counts_dev, void* stream) {
    SNNB_REQUIRE(m, "snnb_model_detect_rois: null model");
    SNNB_CUDA_OK(cudaSetDevice(m->core->ctx->device));
    return m->core->detectRois(frames, num_frames, rois_dev, count_dev, rows_dev, max_rows, counts_dev, static_cast<cudaStream_t>(stream));
}
int snnb_model_detect_rois_list(snnb_model* m, const snnb_frame_list* frames, const snnb_roi* rois_dev, const int* count_dev, float* rows_dev, int max_rows,
                                int* counts_dev, void* stream) {
    SNNB_REQUIRE(m, "snnb_model_detect_rois_list: null model");
    SNNB_CUDA_OK(cudaSetDevice(m->core->ctx->device));
    return m->core->detectRoisList(frames, rois_dev, count_dev, rows_dev, max_rows, counts_dev, static_cast<cudaStream_t>(stream));
}
int snnb_model_transform_frame_list(snnb_model* m, const snnb_frame_list* frames, const snnb_frame_out_list* out, void* stream) {
    SNNB_REQUIRE(m, "snnb_model_transform_frame_list: null model");
    SNNB_CUDA_OK(cudaSetDevice(m->core->ctx->device));
    return m->core->transformFrameList(frames, out, static_cast<cudaStream_t>(stream));
}
int snnb_model_transform_luma_list(snnb_model* m, const snnb_frame_list* frames, const snnb_frame_out_list* out, void* stream) {
    SNNB_REQUIRE(m, "snnb_model_transform_luma_list: null model");
    SNNB_CUDA_OK(cudaSetDevice(m->core->ctx->device));
    return m->core->transformLumaList(frames, out, static_cast<cudaStream_t>(stream));
}
int snnb_model_segment_frame_list(snnb_model* m, const snnb_frame_list* frames, int luma, const snnb_labels_list* out, void* stream) {
    SNNB_REQUIRE(m, "snnb_model_segment_frame_list: null model");
    SNNB_CUDA_OK(cudaSetDevice(m->core->ctx->device));
    return m->core->segmentFrameList(frames, luma != 0, out, static_cast<cudaStream_t>(stream));
}
int snnb_model_set_batch(snnb_model* m, int n) {
    SNNB_REQUIRE(m, "snnb_model_set_batch: null model");
    return m->core->setBatch(n);
}
int snnb_model_set_count_batches(snnb_model* m, const int* sizes, int num_sizes) {
    SNNB_REQUIRE(m, "snnb_model_set_count_batches: null model");
    SNNB_CUDA_OK(cudaSetDevice(m->core->ctx->device));
    return m->core->setCountBatches(sizes, num_sizes);
}
int snnb_model_set_input(snnb_model* m, int idx, const float* host_input) {
    SNNB_REQUIRE(m, "snnb_model_set_input: null model");
    SNNB_CUDA_OK(cudaSetDevice(m->core->ctx->device));
    return m->core->setInput(idx, host_input);
}
int snnb_model_forward(snnb_model* m) {
    SNNB_REQUIRE(m, "snnb_model_forward: null model");
    SNNB_CUDA_OK(cudaSetDevice(m->core->ctx->device));
    return m->core->forward();
}
int snnb_model_get_output(snnb_model* m, int idx, float* host_output, size_t cap) {
    SNNB_REQUIRE(m, "snnb_model_get_output: null model");
    SNNB_CUDA_OK(cudaSetDevice(m->core->ctx->device));
    return m->core->getOutput(idx, host_output, cap);
}
int snnb_model_layer_output(snnb_model* m, int layer, float* host, size_t cap) {
    SNNB_REQUIRE(m, "snnb_model_layer_output: null model");
    SNNB_CUDA_OK(cudaSetDevice(m->core->ctx->device));
    return m->core->layerOutput(layer, host, cap);
}
int snnb_model_dump_outputs(snnb_model* m, const char* dir) {
    SNNB_REQUIRE(m && dir, "snnb_model_dump_outputs: null argument");
    SNNB_CUDA_OK(cudaSetDevice(m->core->ctx->device));
    return m->core->dumpOutputs(dir);
}
int snnb_model_time_layers(snnb_model* m, float* times_ms, int capacity) {
    SNNB_REQUIRE(m && times_ms && capacity >= (int) m->core->layers.size(), "snnb_model_time_layers: bad argument");
    SNNB_CUDA_OK(cudaSetDevice(m->core->ctx->device));
    std::vector<float> ms;
    if (m->core->timeLayers(ms)) return 1;
    for (size_t i = 0; i < ms.size(); ++i) times_ms[i] = ms[i];
    return 0;
}
int snnb_model_launches_per_forward(const snnb_model* m) { return m ? m->core->launchesPerForward : -1; }
int snnb_model_layer_kernel(const snnb_model* m, int layer, char* name, int name_cap) {
    SNNB_REQUIRE(m && name && layer >= 0 && layer < (int) m->core->layers.size(), "snnb_model_layer_kernel: bad argument");
    copyStr(name, name_cap, layer < (int) m->core->layerKernels.size() ? m->core->layerKernels[layer] : std::string());
    return 0;
}

int snnb_model_get_boxes(snnb_model* m, int n, float* rows6, int max_rows, int* count) {
    SNNB_REQUIRE(m && count, "snnb_model_get_boxes: null argument");
    SNNB_REQUIRE(n >= 0 && n < (int) m->core->boxes.size(), "snnb_model_get_boxes: no detections for image %d (model has no YOLO layer, or run() not called)", n);    const auto& rows = m->core->boxes[n].rows;
    int k            = 0;
    for (; k < (int) rows.size() && k < max_rows && k < 100; ++k)
        for (int j = 0; j < 6; ++j) rows6[k * 6 + j] = rows[k][j];
    *count = k;
    return 0;
}

int snnb_model_weight_arena(snnb_model* m, void** device_ptr, size_t* bytes) {
    SNNB_REQUIRE(m && device_ptr && bytes, "snnb_model_weight_arena: null argument");
    *device_ptr = m->core->arena;
    *bytes      = m->core->arenaBytes;
    return 0;
}

// ---- the one collective: ncclBroadcast of the packed weight arena (NCCL resolved at run time, see snnb.h) ----
namespace {
struct NcclApi {
    struct Id { // ncclUniqueId: 128 opaque bytes, passed BY VALUE to ncclCommInitRank
        char b[128];
    };
    typedef int (*GetUniqueId)(void*);
    typedef int (*CommInitRank)(void**, int, Id, int);
    typedef int (*Broadcast)(const void*, void*, size_t, int, int, void*, cudaStream_t);
    typedef int (*CommDestroy)(void*);
    typedef const char* (*GetErrorString)(int);
    GetUniqueId getUniqueId = nullptr;
    CommInitRank commInitRank = nullptr;
    Broadcast broadcast = nullptr;
    CommDestroy commDestroy = nullptr;
    GetErrorString errorString = nullptr;
    bool ok = false;
};
NcclApi& nccl() {
    static NcclApi api;
    static bool tried = false;
    if (!tried) {
        tried = true;
        void* h = RTLD_DEFAULT; // the host process's own NCCL first (PyTorch bundles one): the communicator must live in ONE library
        if (!dlsym(h, "ncclBroadcast")) h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
        if (h) {
            api.getUniqueId  = (NcclApi::GetUniqueId) dlsym(h, "ncclGetUniqueId");
            api.commInitRank = (NcclApi::CommInitRank) dlsym(h, "ncclCommInitRank");
            api.broadcast    = (NcclApi::Broadcast) dlsym(h, "ncclBroadcast");
            api.commDestroy  = (NcclApi::CommDestroy) dlsym(h, "ncclCommDestroy");
            api.errorString  = (NcclApi::GetErrorString) dlsym(h, "ncclGetErrorString");
            api.ok           = api.getUniqueId && api.commInitRank && api.broadcast && api.commDestroy;
        }
    }
    return api;
}
const char* ncclErr(int rc) { return nccl().errorString ? nccl().errorString(rc) : "?"; }
} // namespace

struct snnb_comm {
    snnb_context* ctx = nullptr;
    void* comm        = nullptr;
    int rank = 0, world = 1;
};

int snnb_nccl_unique_id(unsigned char id128[128]) {
    SNNB_REQUIRE(id128, "snnb_nccl_unique_id: null argument");
    SNNB_REQUIRE(nccl().ok, "snnb_nccl_unique_id: NCCL (libnccl.so.2) is not available in this process");
    const int rc = nccl().getUniqueId(id128);
    SNNB_REQUIRE(rc == 0, "ncclGetUniqueId failed: %s", ncclErr(rc));
    return 0;
}
int snnb_nccl_comm_create(snnb_context* ctx, int rank, int world_size, const unsigned char id128[128], snnb_comm** out) {
    SNNB_REQUIRE(ctx && id128 && out && world_size >= 1 && rank >= 0 && rank < world_size, "snnb_nccl_comm_create: bad argument");
    SNNB_REQUIRE(nccl().ok, "snnb_nccl_comm_create: NCCL (libnccl.so.2) is not available in this process");
    SNNB_CUDA_OK(cudaSetDevice(ctx->device));
    NcclApi::Id id;
    memcpy(id.b, id128, 128);
    auto* c  = new snnb_comm();
    c->ctx = ctx, c->rank = rank, c->world = world_size;
    const int rc = nccl().commInitRank(&c->comm, world_size, id, rank);
    if (rc != 0) {
        delete c;
        set_error("ncclCommInitRank(rank %d of %d) failed: %s", rank, world_size, ncclErr(rc));
        return 1;
    }
    *out = c;
    return 0;
}
int snnb_nccl_comm_destroy(snnb_comm* comm) {
    if (!comm) return 0;
    if (comm->comm && nccl().ok) nccl().commDestroy(comm->comm);
    delete comm;
    return 0;
}
int snnb_bcast_weights(snnb_model* m, snnb_comm* comm, int root) {
    SNNB_REQUIRE(m && comm && root >= 0 && root < comm->world, "snnb_bcast_weights: bad argument");
    SNNB_REQUIRE(m->core->ctx == comm->ctx, "snnb_bcast_weights: the communicator was created on another context");
    SNNB_CUDA_OK(cudaSetDevice(comm->ctx->device));
    // in place: rank `root` sends its arena, everyone else receives into theirs (all ranks packed the same layout)
    const int rc = nccl().broadcast(m->core->arena, m->core->arena, m->core->arenaBytes, /* ncclUint8 */ 1, root, comm->comm, comm->ctx->stream);
    SNNB_REQUIRE(rc == 0, "ncclBroadcast(%zu bytes) failed: %s", m->core->arenaBytes, ncclErr(rc));
    return 0;
}

} // extern "C"
