/*
 * snnb.h — C-ABI of libsnn_b200.so: the H100 (sm_90a) backend for ShaderNN's operator / graph API.
 *
 * This is the drop-in boundary (SURVEY.md §8b): plain C, opaque handles, plain pointers and sizes,
 * `int` status (0 = ok, non-zero = error, message via snnb_last_error()), never throws or aborts
 * across the boundary, no torch types. Everything launches on the context's CUDA stream; calls are
 * asynchronous unless stated. One context per device; no internal threads.
 *
 * Each entry point names the reference interface it replaces (paths relative to the reference repo
 * inferenceengine/shadernn @ 6f3fc8b1). INTEGRATION.md shows the C++ glue a ShaderNN maintainer adds
 * (GpuBackendType::CUDA -> CudaBackend : dp::DeviceBackend, CudaRenderPass : dp::RenderPass).
 *
 * Tensor layout at this boundary: host fp32, either NHWC (N added — the reference is N==1) or the
 * reference's own texture layout "C4HW4" (core/inc/snn/imageTexture.h; element (x,y,c) at
 * (((c/4)*H + y)*W + x)*4 + c%4, demo/common/shaderUnitTest.cpp:87-131). Device storage is private:
 * two fp16 planes (hi, lo = value - hi) in NHWC with the channel pitch padded to 8 — an fp32-faithful
 * (22 significant bits, range +-65504) format that TMA can feed straight to the tensor cores (wgmma, see DESIGN.md).
 */
#ifndef SNNB_H_
#define SNNB_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SNNB_VERSION 100

typedef struct snnb_context snnb_context; /* replaces snn::GpuContext + dp::DeviceBackend (core/src/ic2/backend.h:32-91) */
typedef struct snnb_tensor snnb_tensor;   /* replaces snn::ImageTexture device side (core/inc/snn/imageTexture.h:31-352) */
typedef struct snnb_weights snnb_weights; /* replaces InferencePass::_vecWeights/_vecBias/... (core/src/ic2/inferencepass.h:31-59) */
typedef struct snnb_model snnb_model;     /* replaces snn::MixedInferenceCore (core/inc/snn/core.h:66-146) */
typedef struct snnb_timer snnb_timer;     /* replaces snn::DeviceTimer (core/inc/snn/deviceTimer.h) */

/* Activation ids = the Vulkan host's (core/src/ic2/conv2dVulkan.cpp:57-71). SOFTMAX only for Dense. */
enum { SNNB_ACT_NONE = 0, SNNB_ACT_RELU = 1, SNNB_ACT_RELU6 = 2, SNNB_ACT_TANH = 3, SNNB_ACT_SIGMOID = 4, SNNB_ACT_LEAKY_RELU = 5, SNNB_ACT_SILU = 6, SNNB_ACT_SOFTMAX = 7 };
/* Padding modes = conv2dVulkan.cpp:73-80 (0 = unset: out-of-range taps read 0, same as constant). */
enum { SNNB_PAD_NONE = 0, SNNB_PAD_CONSTANT = 1, SNNB_PAD_REPLICATE = 2, SNNB_PAD_REFLECT = 3 };
/* Kernel selection for convolutions. AUTO picks the tensor-core (wgmma) implicit-GEMM path when the shape allows. TCGEN05_STREAMK also lets the
 * planner cut the K loops of the last partial wave of tiles across all SMs (stream-K; measured slower than whole tiles on ResNet-18's
 * shapes - DESIGN.md 3.4 - so it is not part of AUTO; environment SNNB_SK=1 enables it for every launch). */
enum { SNNB_ALGO_AUTO = 0, SNNB_ALGO_SIMT = 1, SNNB_ALGO_TCGEN05 = 2, SNNB_ALGO_TCGEN05_STREAMK = 3 };
/* Arithmetic / storage precision of the tensor-core convolution path (the reference's counterpart is
 * ShaderGenOptions::preferrHalfPrecision, core/inc/snn/layeroption.h:43: fp32 by default, RGBA16F when set).
 *   FP32X3: activations AND weights as fp16 hi+lo pairs, three fp16 MMAs per product: fp32-class (~22 bits per operand).
 *   FP16W : activations as fp16 hi+lo pairs, weights rounded once to fp16 (<= 2^-12 relative per weight), two MMAs per product.
 *   FP16  : the half-precision storage mode (= the reference's RGBA16F textures): one fp16 plane per tensor and per weight,
 *           one MMA per product, half the bytes. Meets the reference's half-precision tolerance (0.1,
 *           demo/common/testutil.h:1195), NOT the 1e-3 fp32 bar. */
enum { SNNB_PRECISION_FP32X3 = 0, SNNB_PRECISION_FP16W = 1, SNNB_PRECISION_FP16 = 2 };

/* ---- context / errors -------------------------------------------------------------------------------------- */
/* dp::BackendBuilder::build (core/src/ic2/backendBuilder.cpp:28-50) + context creation (core/src/contextFactory.cpp). */
int snnb_context_create(int device, snnb_context** out);
int snnb_context_destroy(snnb_context* ctx);
/* DeviceBackend::sync (backend.h:60; vulkanBackend.cpp:97-106 QueueSubmitAndWait). */
int snnb_sync(snnb_context* ctx);
/* The cudaStream_t everything is launched on (as void*). */
void* snnb_context_stream(snnb_context* ctx);
/* Thread-local message of the last failing call (replaces SNN_RIP / SNN_LOGE text, core/inc/snn/utils.h:57-62). */
const char* snnb_last_error(void);
/* Number of kernels this library has launched on the context since creation (bench.py's gpu_launches). */
uint64_t snnb_launch_count(snnb_context* ctx);
int snnb_version(void);
/* Default precision of per-operator convolution launches on this context (SNNB_PRECISION_FP32X3 or _FP16W; models carry
 * their own in snnb_model_options). */
int snnb_context_set_precision(snnb_context* ctx, int precision);

/* ---- tensors ------------------------------------------------------------------------------------------------ */
/* ImageTextureAllocator / ImageTexture::resetTexture + upload()/download() (imageTexture.h:60-147). */
int snnb_tensor_alloc(snnb_context* ctx, int n, int h, int w, int c, snnb_tensor** out);
int snnb_tensor_free(snnb_tensor* t);
int snnb_tensor_dims(const snnb_tensor* t, int* n, int* h, int* w, int* c);
int snnb_tensor_upload_nhwc(snnb_context* ctx, snnb_tensor* t, const float* host_nhwc);   /* synchronous */
int snnb_tensor_download_nhwc(snnb_context* ctx, const snnb_tensor* t, float* host_nhwc); /* synchronous */
/* Reference texture layout, per image: [ceil(C/4)][H][W][4]; images concatenated over N. */
int snnb_tensor_upload_c4hw4(snnb_context* ctx, snnb_tensor* t, const float* host_c4hw4);
int snnb_tensor_download_c4hw4(snnb_context* ctx, const snnb_tensor* t, float* host_c4hw4);
/* Debug dump in the reference's .dump format: 32-byte ASCII header "W H D C" + [D][H][W][4] fp32
 * (core/src/image.cpp:216-245). One file per image when N > 1 ("<path>.n<i>"). */
int snnb_tensor_dump(snnb_context* ctx, const snnb_tensor* t, const char* path);

/* ---- weights: fold + pack at load time ------------------------------------------------------------------------ */
/* Conv2DDesc (core/src/ic2/conv2d.h) + Conv2DLayer::getPaddingOffset (conv2d.cpp:39-74). pad_x/pad_y are the
 * shader's uPadx/uPady (NB the reference feeds offsets[0]=top as x and offsets[2]=left as y, conv2dVulkan.cpp:183-184). */
typedef struct {
    int in_channels, out_channels, kernel, stride;
    int pad_x, pad_y, pad_mode;
    int activation;
    float leaky_alpha;
    int algo; /* SNNB_ALGO_* */
} snnb_conv_desc;

/* Replaces Conv2DLayer::oihw2hwo4i4 (conv2d.cpp:76-100) + the BN/bias buffers of conv2dVulkan.cpp:110-152.
 * w_oihw: OC*IC*k*k (modelparser.cpp:641-657). bias / bn_* may be NULL. BN (eps 1e-3, sqrt clamp 1e-4,
 * vk_conv2d.comp:277-288) is folded into the packed weights and bias here. */
int snnb_weights_pack_conv2d(snnb_context* ctx, const snnb_conv_desc* d, const float* w_oihw, const float* bias, const float* bn_gamma,
                             const float* bn_beta, const float* bn_mean, const float* bn_var, snnb_weights** out);
/* Replaces SeparableConv2DLayer::oihw2hwo4i4 (separableconvolution.cpp:88-111). w_chw: C*k*k ([C][kh][kw], the
 * parser's mats, modelparser.cpp:827-850). in_channels == out_channels == C. */
int snnb_weights_pack_depthwise(snnb_context* ctx, const snnb_conv_desc* d, const float* w_chw, const float* bias, const float* bn_gamma,
                                const float* bn_beta, const float* bn_mean, const float* bn_var, snnb_weights** out);
/* Dense (denselayer.cpp:27-54): kernel is the flat JSON array viewed [out][in] (cpulayer.h:162). */
int snnb_weights_pack_dense(snnb_context* ctx, int n_in, int n_out, const float* kernel_out_in, const float* bias, snnb_weights** out);
/* Per-channel vectors (BatchNormalization: gamma,beta,mean,var; InstanceNorm: gamma,beta). Any may be NULL (defaults 1,0,0,1). */
int snnb_weights_pack_channels(snnb_context* ctx, int channels, const float* gamma, const float* beta, const float* mean, const float* var,
                               snnb_weights** out);
int snnb_weights_free(snnb_weights* w);

/* ---- operator launches (one call == one RenderPass::run, core/src/ic2/renderpass.h:64) ------------------------- */
/* Conv2D k x k incl. 1x1 (shadertemplate_vk_conv2d.comp:148-347, vk_conv2d_1x1.comp:68-211). `residual` (may be
 * NULL) is added before the activation: the fused form of Conv2D -> Add(+act) (vk_add.comp:41-90). */
int snnb_conv2d_launch(snnb_context* ctx, const snnb_conv_desc* d, const snnb_weights* w, const snnb_tensor* in, const snnb_tensor* residual,
                       snnb_tensor* out);
/* Depthwise k x k (shadertemplate_vk_depthwise.comp:64-139). */
int snnb_depthwise_launch(snnb_context* ctx, const snnb_conv_desc* d, const snnb_weights* w, const snnb_tensor* in, snnb_tensor* out);
/* MaxPooling2D / AveragePooling2D (vk_maxpool2d.comp:42-71, vk_avgpool2d.comp:42-69; window origin o*stride). */
int snnb_maxpool_launch(snnb_context* ctx, int kernel, int stride, const snnb_tensor* in, snnb_tensor* out);
int snnb_avgpool_launch(snnb_context* ctx, int kernel, int stride, const snnb_tensor* in, snnb_tensor* out);
/* Add + activation (vk_add.comp:41-90). */
int snnb_add_launch(snnb_context* ctx, int activation, float leaky_alpha, const snnb_tensor* a, const snnb_tensor* b, snnb_tensor* out);
/* Standalone BatchNormalization + activation (vk_batchnorm.comp:54-69); w from snnb_weights_pack_channels. */
int snnb_batchnorm_launch(snnb_context* ctx, const snnb_weights* w, int activation, float leaky_alpha, const snnb_tensor* in, snnb_tensor* out);
/* Standalone activation (vk_activation.comp:41-85). */
int snnb_activation_launch(snnb_context* ctx, int activation, float leaky_alpha, const snnb_tensor* in, snnb_tensor* out);
/* Dense + activation incl. softmax (cpulayer.h:136-261; GPU twin vk_dense.comp:53-83). in: [N,1,1,n_in] (or any
 * [N,H,W,C] with H*W*C == n_in, consumed in HWC order = CPU Flatten, cpulayer.h:94-115). out: [N,1,1,n_out]. */
int snnb_dense_launch(snnb_context* ctx, const snnb_weights* w, int activation, float leaky_alpha, const snnb_tensor* in, snnb_tensor* out);
/* Softmax over channels per pixel (cpulayer.h:175-191) and classifier index argmax+1 (core.cpp:228-233), per image. */
int snnb_softmax_launch(snnb_context* ctx, const snnb_tensor* in, snnb_tensor* out);
int snnb_argmax1(snnb_context* ctx, const snnb_tensor* in, int* host_idx_1based); /* synchronous; in: [N,1,1,C] */
/* Flatten in HWC order (cpulayer.h:94-115): [N,H,W,C] -> [N,1,1,H*W*C]. */
int snnb_flatten_launch(snnb_context* ctx, const snnb_tensor* in, snnb_tensor* out);
/* Concatenate along channels (vk_concat.comp:39-52). */
int snnb_concat_launch(snnb_context* ctx, const snnb_tensor* a, const snnb_tensor* b, snnb_tensor* out);
/* UpSampling2D nearest / bilinear (vk_upsampling2d_nearest.comp:43-64, _bilinear.comp:43-86). */
int snnb_upsample_launch(snnb_context* ctx, float scale, int bilinear, const snnb_tensor* in, snnb_tensor* out);
/* Pad constant/replicate/reflect (vk_pad.comp:42-70). */
int snnb_pad_launch(snnb_context* ctx, int pad_x, int pad_y, int pad_mode, const snnb_tensor* in, snnb_tensor* out);
/* InstanceNorm (+act), biased variance, eps 1e-5 (vk_instancenorm.comp:53-175). */
int snnb_instancenorm_launch(snnb_context* ctx, const snnb_weights* w, int activation, float leaky_alpha, const snnb_tensor* in, snnb_tensor* out);
/* Subpixel: depth_to_space(r) + tanh, always (vk_subpixel.comp:43-70, fs_subpixel.glsl:41). */
int snnb_subpixel_launch(snnb_context* ctx, int r, const snnb_tensor* in, snnb_tensor* out);

/* ---- device timers (DeviceBackend::createDeviceTimer, backend.h:79; core.cpp:140-152) --------------------------- */
int snnb_timer_create(snnb_context* ctx, snnb_timer** out);
int snnb_timer_start(snnb_timer* t);
int snnb_timer_stop(snnb_timer* t);
int snnb_timer_elapsed_ms(snnb_timer* t, float* ms); /* synchronises on the stop event */
int snnb_timer_destroy(snnb_timer* t);

/* ---- launch capture for backend-level integration -------------------------------------------------------------
 * A DeviceBackend built on the per-operator calls (INTEGRATION.md, depth B) records its stage loop once and replays it:
 * everything launched on the context between capture_begin and capture_end becomes one CUDA graph (the counterpart of
 * recording the reference's single command buffer, vulkanBackend.cpp:97-106). Run the same launches eagerly once before
 * capturing: lazily created resources (tensor-map encoder, split-K scratch) must exist, because allocation is illegal
 * while capturing. Tensors and weights referenced by the graph must outlive it. */
typedef struct snnb_graph snnb_graph;
int snnb_graph_capture_begin(snnb_context* ctx);
int snnb_graph_capture_end(snnb_context* ctx, snnb_graph** out);
int snnb_graph_launch(snnb_graph* g); /* asynchronous on the context's stream */
int snnb_graph_destroy(snnb_graph* g);

/* ---- whole-model engine: dp::loadFromJsonModel + generateInferenceGraph + MixedInferenceCore ------------------- */
typedef struct {
    int batch;          /* images per run() on this GPU (the reference is fixed at 1, inferencegraph.h:58-64) */
    int input_width;    /* ShaderGenOptions::desiredInput (layeroption.h:30); 0 = use the JSON InputLayer's */
    int input_height;
    int conv_algo;      /* SNNB_ALGO_*: AUTO by default */
    int use_cuda_graph; /* replay the captured forward pass instead of re-launching kernels */
    int fuse;           /* graph-level fusion passes (conv+add+act, pad->conv); 0 keeps 1 kernel per reference layer */
    int precision;      /* SNNB_PRECISION_*; FP16 = the reference's preferrHalfPrecision (layeroption.h:43) */
} snnb_model_options;

/* MixedInferenceCore::create(ctx, modelFileName, options) (core.h:115-116) = dp::loadFromJsonModel (dp.cpp:115-167:
 * ModelParser ctor modelparser.cpp:210-258 incl. the sidecar .bin next to the JSON) + generateInferenceGraph
 * (dp.cpp:432-640) + init (core.cpp:294-410) + weight fold/pack/upload. */
int snnb_model_load_json(snnb_context* ctx, const char* json_path, const snnb_model_options* opt, snnb_model** out);
int snnb_model_destroy(snnb_model* m);
int snnb_model_num_layers(const snnb_model* m);
/* Layer i in JSON order: name "<json file> layer [NN] <Type>" (dp.cpp:135), type string, output dims. */
int snnb_model_layer_info(const snnb_model* m, int i, char* name, int name_cap, char* type, int type_cap, int* n, int* h, int* w, int* c);
int snnb_model_num_inputs(const snnb_model* m);
int snnb_model_num_outputs(const snnb_model* m);
int snnb_model_input_dims(const snnb_model* m, int idx, int* n, int* h, int* w, int* c);
int snnb_model_output_dims(const snnb_model* m, int idx, int* n, int* h, int* w, int* c);
/* MixedInferenceCore::run (core.cpp:97-245), end to end with HOST buffers: H2D of the NHWC fp32 batch, forward,
 * D2H of output 0 (NHWC fp32, out_capacity floats) and, for classifiers (last layer Dense/softmax), the 1-based
 * class index per image (core.cpp:228-233); classes may be NULL. Synchronous. */
int snnb_model_run(snnb_model* m, const float* host_input_nhwc, float* host_output, size_t out_capacity, int* classes_1based);
/* Streaming variant of snnb_model_run for serving loops: submit() enqueues the H2D copy of the batch (on a dedicated copy
 * stream, double-buffered device staging), the forward pass and the D2H copies of output 0 / class indices into the
 * caller's buffers, and returns at once with a ticket; wait(ticket) blocks until that submission's results are in host
 * memory. Up to two submissions may be in flight, so batch i+1's upload overlaps batch i's compute. Host buffers must be
 * pinned for the copies to be asynchronous and must stay untouched until wait() returns. (The reference's run() is
 * strictly synchronous, core.cpp:97-245; this is additive.) */
int snnb_model_submit(snnb_model* m, const float* host_input_nhwc, float* host_output, size_t out_capacity, int* classes_1based, int* ticket);
/* submit() for 8-bit images: host_input is N*H*W*C bytes (NHWC, dense); the device computes (x - mean4[c & 3]) * norm4[c & 3]
 * while converting, i.e. ImageTexture::convertToRGBA32FAndNormalize(means, norms) (core/inc/snn/imageTexture.h:114; per-model
 * constants in demo/common/modelInference.cpp:135-224, e.g. ResNet-18 mean 127.5 norm 1/127.5) without a host pass, and a
 * quarter of the fp32 bytes cross PCIe. */
int snnb_model_submit_u8(snnb_model* m, const uint8_t* host_input_nhwc_u8, const float* mean4, const float* norm4, float* host_output, size_t out_capacity,
                         int* classes_1based, int* ticket);
/* Image in, image (or tensor) out, all pre/post-processing on the device (SURVEY §8 f-N3): the 8-bit input may have ANY size - it is
 * resized to the model's input with the linear or nearest filter exactly as ImageTexture::resize does (imageTexture.h:137,
 * shadertemplate_vk_resize.comp:42-61: output texel centres sampled from the source) and normalised in the same kernel; the result comes
 * back either as fp32 (output_f32) or as an 8-bit image, clamp(round(v * out_scale + out_offset), 0, 255) (style transfer: scale 1;
 * a tanh output: 127.5 / 127.5). Same ticket / wait protocol as snnb_model_submit. */
typedef struct {
    const uint8_t* input_u8; /* N * src_height * src_width * C bytes, NHWC, dense */
    int src_height, src_width;
    int linear_filter;       /* 1 = linear (the reference's default), 0 = nearest */
    float mean4[4], norm4[4];
    float* output_f32;       /* exactly one of output_f32 / output_u8 may be non-NULL (both NULL: no output copy) */
    size_t output_capacity;  /* elements */
    uint8_t* output_u8;
    float out_scale, out_offset;
    int* classes_1based;     /* classifiers only, may be NULL */
} snnb_image_io;
int snnb_model_submit_image(snnb_model* m, const snnb_image_io* io, int* ticket);
int snnb_model_wait(snnb_model* m, int ticket);
/* Inputs and outputs that already live in device memory, ordered on the caller's CUDA stream: the counterpart of attaching GPU images
 * to the model (ModelInput / ModelOutput attach(), genericModelProcessorVulkan.cpp:112-121, styleTransferProcessorGL.cpp:175-181;
 * RunParameters::inputImages / outputImages, core/inc/snn/core.h:78-80) and run(). Nothing crosses PCIe and nothing waits on the host.
 *
 * A buffer is `data`: device (or managed) memory of the model's device, dense in `layout`, the batch x H x W x C of its tensor
 * (N x C x H x W for NCHW), aligned to its element size. U8 inputs are normalised as (x - mean4[c & 3]) * norm4[c & 3], exactly as
 * snnb_model_submit_u8; U8 outputs are clamp(round(v * scale + offset), 0, 255), exactly as snnb_image_io.output_u8; F16 outputs are
 * the fp32 values rounded to nearest. The other fields are ignored. */
enum { SNNB_DTYPE_F32 = 0, SNNB_DTYPE_F16 = 1, SNNB_DTYPE_U8 = 2 };
enum { SNNB_LAYOUT_NHWC = 0, SNNB_LAYOUT_NCHW = 1 };
typedef struct {
    void* data;
    int dtype, layout;        /* SNNB_DTYPE_*, SNNB_LAYOUT_* */
    float mean4[4], norm4[4]; /* U8 inputs only */
    float scale, offset;      /* U8 outputs only */
} snnb_device_buffer;
/* - inputs: num_inputs must equal snnb_model_num_inputs(); inputs[i] feeds InputLayer i in "inputIndex" order (so a model with several
 *   inputs can be fed here, while run() / submit() feed input 0 only).
 * - outputs: outputs[j] receives model output j, for j < num_outputs <= snnb_model_num_outputs(); an entry with data == NULL is skipped,
 *   and num_outputs may be 0 (classes only).
 * - classes_1based_dev: NULL, or device int32[batch] that receives arg-max + 1 per image (core.cpp:228-233). An error for a model that
 *   is not a classifier.
 * - stream: a cudaStream_t of the model's device, or NULL for the context's stream. To order against a default stream, pass
 *   cudaStreamLegacy or cudaStreamPerThread, not NULL. The call returns without waiting for the GPU: work enqueued on `stream` before
 *   the call happens before the inputs are read, and work enqueued on `stream` after it sees the outputs. The model's work itself runs
 *   on the context's stream, behind two events per model (the caller's stream -> the context's stream -> the caller's stream), so calls
 *   from different streams, and calls mixed with run() / submit(), are serialised on the model's tensors. A stream that is being
 *   captured is refused: capturing this call into the caller's CUDA graph is not supported.
 * - The batch is the loaded batch. A model whose output 0 is a YOLO layer is refused: its detections come through
 *   snnb_model_detect_device below, or the host paths (run() / submit() + snnb_model_get_boxes).
 * Every argument is checked on the host before anything is enqueued: null pointers, unknown dtype or layout, the input count, buffers
 * that cudaPointerGetAttributes does not report as device or managed memory of the context's device, and misaligned buffers are errors
 * (snnb_last_error()) with no work enqueued. A buffer's size cannot be checked: it must hold its tensor's elements. Cost beyond the
 * forward pass: one kernel launch per input, one per output and one for the classes. */
int snnb_model_run_device(snnb_model* m, const snnb_device_buffer* inputs, int num_inputs, const snnb_device_buffer* outputs, int num_outputs,
                          int* classes_1based_dev, void* stream);
/* Detectors on device-resident inputs: the forward pass, then YOLO decode + score sort + NMS (yololayer.cpp:56-226) on the device.
 * inputs: exactly as snnb_model_run_device. rows_dev: float32 [batch][max_rows][6] {class, score, x, y, w, h}, rows past an image's
 * count are zero; counts_dev: int32 [batch], min(kept boxes, max_rows, 100) per image, as snnb_model_get_boxes counts them.
 * 1 <= max_rows <= 100. Same stream contract, fences and host-side argument checks as snnb_model_run_device; refused for a model
 * without a YOLO output. Does not touch the host detections that snnb_model_get_boxes returns.
 * The rows are those of the host paths, in the same order, with one difference in arithmetic: the device uses the correctly rounded
 * exponential, (float) exp((double) x), where the host calls the C library's expf, so a score or coordinate can differ in its last
 * bit or two. Cost beyond the forward pass: one kernel launch per input, one memset and three decode kernels. */
int snnb_model_detect_device(snnb_model* m, const snnb_device_buffer* inputs, int num_inputs, float* rows_dev, int max_rows,
                             int* counts_dev, void* stream);
/* Device-resident 8-bit video frames of any size (NVDEC's NV12, nvJPEG's I420, a camera's NV21, an RGBA image) into input 0 of a
 * model with exactly one input of 1 to 4 channels: the reference's camera path NativeFrameProvider::copyImageData = nv12ToRgba8 /
 * nv21ToRgba8 / i420ToRgba8 (core/src/image.cpp:1076-1136, libyuv's 6-bit fixed-point YuvPixel, BT.601 limited range) ->
 * ImageTexture::resize -> convertToRGBA32FAndNormalize, fused into ONE kernel that writes the model input. Model channel c is RGBA
 * component c. Per output pixel: the source taps of ImageTexture::resize (snnb_image_io; when the frame has the model's size, the
 * pixel itself), each converted to RGBA8 exactly as libyuv does, pixel (x, y) using chroma sample (x / 2, y / 2); then the same
 * interpolation and normalisation as snnb_model_submit_image. The model input is therefore bit-identical to snnb_model_submit_image
 * fed libyuv's RGBA8 image (its first C components). */
enum { SNNB_FRAME_NV12 = 0, SNNB_FRAME_NV21 = 1, SNNB_FRAME_I420 = 2, SNNB_FRAME_RGBA8 = 3 };
enum { SNNB_YUV_BT601 = 0 /* libyuv kYuvI601Constants: the reference's nv12ToRgba8 */, SNNB_YUV_BT709 = 1 /* kYuvH709Constants */ };
typedef struct {
    int format, matrix;          /* SNNB_FRAME_*, SNNB_YUV_* (matrix ignored for RGBA8) */
    int width, height;           /* frame size, any >= 1 (odd allowed: chroma is ceil(w/2) x ceil(h/2), as libyuv) */
    const uint8_t* plane[3];     /* NV12/NV21: Y, UV|VU; I420: Y, U, V; RGBA8: RGBA. Device memory of the model's device */
    int pitch[3];                /* bytes per row, >= the row's bytes */
    long long image_stride[3];   /* bytes from image n to image n+1 of the batch, per plane */
    int linear_filter;           /* as snnb_image_io */
    float mean4[4], norm4[4];    /* (x - mean4[c]) * norm4[c] on the RGBA component c */
} snnb_frames;
/* snnb_model_run_device / snnb_model_detect_device with `frames` (the loaded batch of them) in place of the input buffers: outputs,
 * classes, rows, counts, the stream contract and the fences are exactly theirs; run_frames refuses YOLO models, detect_frames requires
 * them. Checked on the host before anything is enqueued: format and matrix, width and height >= 1, each pitch >= its row's bytes, each
 * plane device or managed memory of the context's device, a model with one input of <= 4 channels, a stream that is not capturing.
 * A plane's size cannot be checked: it must hold the batch. Cost beyond the forward pass: one kernel launch for the input (1920x1080
 * NV12 to YOLOv3-tiny 416x416 x 16: 50 us, to ResNet-18 224x224 x 32: 30 us; NVIDIA H100 80GB HBM3, 700 W power limit). */
int snnb_model_run_frames(snnb_model* m, const snnb_frames* frames, const snnb_device_buffer* outputs, int num_outputs, int* classes_1based_dev,
                          void* stream);
int snnb_model_detect_frames(snnb_model* m, const snnb_frames* frames, float* rows_dev, int max_rows, int* counts_dev, void* stream);
/* Image-to-image models (style transfer, super-resolution) from device frames to device frames: snnb_model_run_frames' input, the
 * forward pass, then output 0 written as the loaded batch of 8-bit frames of any size, for an encoder (NV12) or a display (RGBA8). It
 * replaces a U8 output followed by a resize, an RGB -> YUV conversion and a pack in the caller's own code. The reference's path is
 * the same: the output goes to an RGBA8 texture, ImageTexture::resize, then rgba8ToNv12 / rgba8ToNv21 / rgba8ToI420
 * (core/src/image.cpp:1051-1100 = libyuv ABGRToNV12 / ABGRToNV21 / ABGRToI420). Every output byte, for image n of output 0
 * (H_o x W_o x C, C = 1, 3 or 4):
 *   1. M, an RGBA8 image of the model's size: each component clamp(rint(v * scale + offset), 0, 255), exactly the U8 output of
 *      snnb_model_run_device. C = 4: RGBA; C = 3: RGB, A = 255; C = 1: R = G = B = that value, A = 255 (a luminance or a mask).
 *   2. F = ImageTexture::resize of M to width x height (the taps of snnb_image_io; F = M at equal sizes). Linear: top = p00 + ax * (p01
 *      - p00), bot = p10 + ax * (p11 - p10), v = top + ay * (bot - top) in IEEE float32 with every operation rounded on its own, then
 *      rint(v).
 *   3. RGBA8: F. NV12 / NV21 / I420: libyuv's ABGRToNV12 / ABGRToNV21 / ABGRToI420 of F with its portable C rows: BT.601 limited range,
 *      Y = (66 R + 129 G + 25 B + 0x1080) >> 8; each chroma sample averages its 2 x 2 block as (a + b + c + d) >> 2 (an odd last column
 *      (a + b) >> 1 over its two rows, an odd last row paired with itself), U = (112 B - 74 G - 38 R + 0x8080) >> 8, V = (112 R - 94 G -
 *      18 B + 0x8080) >> 8. An encoder fed these frames must signal BT.601 limited range.
 * Bytes of a plane outside its rows (pitch padding, gaps between planes and images) are not written. `out` may alias `frames` (an
 * in-place filter of a decoder surface): the output is written after the forward pass, in stream order. */
typedef struct {
    int format;                 /* SNNB_FRAME_*; the YUV formats are BT.601 limited range */
    int width, height;          /* any >= 1 (odd allowed: chroma is ceil(w/2) x ceil(h/2), as libyuv) */
    uint8_t* plane[3];          /* NV12/NV21: Y, UV|VU; I420: Y, U, V; RGBA8: RGBA. Device memory of the model's device */
    int pitch[3];               /* bytes per row, >= the row's bytes */
    long long image_stride[3];  /* bytes from image n to image n+1, per plane */
    int linear_filter;          /* resize filter, as snnb_image_io */
    float scale, offset;        /* model output -> 8 bits, exactly as the U8 output of snnb_model_run_device */
} snnb_frames_out;
/* frames: exactly as snnb_model_run_frames, with the same checks. Also checked on the host before anything is enqueued: out's format,
 * width and height >= 1, each used pitch >= its row's bytes, each used plane device or managed memory of the context's device, and an
 * output 0 of 1, 3 or 4 channels that is not a YOLO layer. Stream contract and fences: those of snnb_model_run_device. Cost beyond the
 * forward pass: one kernel launch for the input and one for the output (Candy 720x720 x 8 to 1920x1080 NV12: 263 us; NVIDIA H100 80GB
 * HBM3, 400 W power limit). */
int snnb_model_transform_frames(snnb_model* m, const snnb_frames* frames, const snnb_frames_out* out, void* stream);
/* Luma models (ESPCN-style super-resolution; a denoiser, deblocker or sharpener of Y) from device frames to device frames: the Y plane
 * feeds a model whose one input has 1 channel, output 0 (1 channel) becomes the Y plane of `out`, and the source chroma is resized
 * beside it, so the colour of the video is kept. It replaces a copy of the Y plane, a U8 run, a chroma resize and a pack in the
 * caller's own code. No colour conversion happens. Every byte, for image n of the loaded batch:
 *   1. Model input: (Y' - mean4[0]) * norm4[0], Y' = ImageTexture::resize of the Y plane to the model's size with frames.linear_filter
 *      (the taps of snnb_image_io; the byte itself at equal sizes). Bit-identical to snnb_model_submit_image fed the Y planes as an
 *      N x H x W x 1 8-bit image. frames.matrix is checked as snnb_model_run_frames checks it and not used.
 *   2. Y plane: M = clamp(rint(v * scale + offset), 0, 255) of output 0 (exactly the U8 output of snnb_model_run_device), then
 *      ImageTexture::resize of M to out.width x out.height with out.linear_filter, blended and rounded as step 2 of
 *      snnb_model_transform_frames (Y = M at equal sizes). This is the byte snnb_model_transform_frames writes as R for that output.
 *   3. Chroma: U and V each ImageTexture::resize of the source's U and V plane, plane to plane, from ceil(W/2) x ceil(H/2) to
 *      ceil(width/2) x ceil(height/2), with out.linear_filter and the same taps, blend and rint as step 2 (a copy at equal chroma sizes).
 *      Resizing the planes on their own, as libyuv's I420Scale does, keeps each sample sited at the centre of its 2 x 2 block.
 * frames.format and out.format are NV12, NV21 or I420 and may differ; RGBA8 is refused on either side. Bytes of a plane outside its rows
 * (pitch padding, gaps between planes and images) are not written. Aliasing: the Y plane is written after the forward pass, but the
 * output kernel reads the source chroma while it writes. So `out` may be `frames` itself (same format, size, planes, pitches and image
 * strides: an in-place luma filter); otherwise no out plane may overlap a source chroma plane. Checked on the host before anything is
 * enqueued: everything snnb_model_transform_frames checks, a model input and an output 0 of exactly 1 channel, and the overlap rule on
 * each plane's bytes, plane + (N - 1) * image_stride + (rows - 1) * pitch + its row's bytes. Stream contract and fences: those of
 * snnb_model_run_device. Cost beyond the forward pass: one kernel launch for the input and one for the output (ESPCN 1920x1080 x 1
 * from 1920x1080 NV12 to 3840x2160 NV12: 24 us and 106 us; NVIDIA H100 80GB HBM3, 400 W power limit). */
int snnb_model_transform_luma(snnb_model* m, const snnb_frames* frames, const snnb_frames_out* out, void* stream);
/* Segmentation models (U-Net, a per-pixel classifier) from device frames to an 8-bit label plane of any size: the class scores of
 * output 0 are resampled to the plane and reduced to one byte per pixel in the same kernel, so neither the upsampled scores nor an
 * arg-max pass ever reach memory. The input is exactly what snnb_model_run_frames feeds (luma == 0), or exactly what
 * snnb_model_transform_luma feeds (luma == 1: the Y plane of NV12 / NV21 / I420 frames into a model input of 1 channel, for grey-input
 * models such as the reference's U-Net). Let T be output 0 (N x h x w x C) with values v = float(hi) + float(lo) (lo absent in FP16
 * storage): bit for bit the F32 output of snnb_model_run_device / snnb_model_run_frames. For label pixel (x, y) of image n:
 *   1. Scores s_c: T[n, y, x, c] when the plane has the output's size; otherwise the taps of ImageTexture::resize of T to width x
 *      height (those of snnb_image_io): nearest takes T at the tap, linear blends the four taps per channel exactly as step 2 of
 *      snnb_model_transform_frames (every + - * rounded on its own, no FMA), on the fp32 scores rather than on 8-bit values.
 *   2. Label: C >= 2: the smallest c whose s_c equals the maximum over the s_c that are not NaN; 0 if every s_c is NaN. C == 1:
 *      1 if s_0 >= threshold, else 0 (NaN gives 0).
 *   3. The label is written at plane + n * image_stride + y * pitch + x. Bytes outside the rows are not written.
 * Checked on the host before anything is enqueued: everything snnb_model_run_frames checks (with luma, also those of
 * snnb_model_transform_luma's input), a non-null out, width and height >= 1, pitch >= width, a plane in device or managed memory of the
 * context's device, and an output 0 that is not a YOLO layer, has a device tensor and has at most 256 channels. A capturing stream is
 * refused. Stream contract and fences: those of snnb_model_run_device. The labels are written after the forward pass and read only the
 * model's tensor, so the plane may overlap the input frames. Cost beyond the forward pass: one kernel launch for the input and one
 * for the labels (U-Net 256x256 x 8 from 1920x1080 NV12 to 1920x1080 labels: 144 us for 1 class, 591 us for 21; NVIDIA H100 80GB
 * HBM3, 700 W power limit). */
typedef struct {
    int width, height;       /* label plane size, any >= 1 */
    uint8_t* plane;          /* device memory of the model's device: one byte per pixel */
    int pitch;               /* bytes per row, >= width */
    long long image_stride;  /* bytes from image n to image n+1 */
    int linear_filter;       /* resampling of the scores: 1 = linear, 0 = nearest (ImageTexture::resize's taps) */
    float threshold;         /* 1-channel outputs only */
} snnb_labels_out;
int snnb_model_segment_frames(snnb_model* m, const snnb_frames* frames, int luma, const snnb_labels_out* out, void* stream);
/* Regions of device frames as the batch: the second stage of a detection pipeline (classify, describe or embed what a detector found)
 * without a host round trip. A region is a pixel rectangle [x, x + width) x [y, y + height) of frame `frame` of the frames given; `row`
 * is carried for the caller (the detection row it came from, or anything) and ignored by the engine. */
typedef struct {
    int frame, row, x, y, width, height;
} snnb_roi;
/* The model's loaded batch B is the number of region slots. rois_dev: device memory holding snnb_roi[B]. count_dev: NULL (all B slots
 * are used) or a device int; slots i < clamp(*count_dev, 0, B) are used. frames: an snnb_frames exactly as snnb_model_run_frames takes
 * it, holding num_frames >= 1 frames (independent of B). A used slot is valid when 0 <= frame < num_frames, width, height >= 1,
 * 0 <= x, x + width <= frames.width, 0 <= y and y + height <= frames.height; the regions live on the device, so this cannot be checked
 * on the host.
 * Slot i, when valid, gets exactly the model input snnb_model_run_frames computes for an RGBA8 frame S_i: S_i is the rectangle cut out of
 * libyuv's RGBA8 image of the whole frame (chroma sited in frame coordinates: pixel (x, y) takes chroma sample (x / 2, y / 2)), then
 * resized as run_frames resizes a frame, with taps clamped to the edges of the region; a region of the model's size is sampled directly.
 * Slots past the count and invalid slots get an all-zero input, and every byte of their outputs and their class is zero (classes are
 * 1-based: 0 = no region). The forward pass runs on the whole batch.
 * Outputs, classes, the stream contract and the fences are those of snnb_model_run_frames; YOLO models are refused (no detection on
 * regions). Checked on the host before anything is enqueued: everything run_frames checks, num_frames >= 1, rois_dev (and count_dev
 * unless NULL) device or managed memory of the context's device, aligned to 4 bytes. Cost beyond run_frames: one kernel launch per
 * output buffer and one for the classes, which clear the slots that hold no region. */
int snnb_model_run_rois(snnb_model* m, const snnb_frames* frames, int num_frames, const snnb_roi* rois_dev, const int* count_dev,
                        const snnb_device_buffer* outputs, int num_outputs, int* classes_1based_dev, void* stream);
typedef struct {
    float min_score; /* rows with score >= min_score are kept */
    int class_id;    /* -1 = any class, else rows of this class only */
    float expand;    /* >= 0: the fraction of w (h) added on each side */
} snnb_roi_select;
/* snnb_model_detect_frames / snnb_model_detect_device rows (rows_dev float32 [num_frames][max_rows][6] {class, score, x, y, w, h},
 * normalised, x, y the top-left corner) and counts (counts_dev int32 [num_frames]) -> regions of frame_width x frame_height frames, for
 * snnb_model_run_rois. One kernel on `stream` (NULL: the context's stream); never synchronises. Rows r < min(counts[n], max_rows) of
 * frame n are visited frame by frame, rows in order (descending score). A row is kept when score >= min_score, class_id is -1 or the
 * row's class, and its rectangle is non-empty. The rectangle, in float32 with every operation rounded on its own (no FMA):
 *   ex = expand * w, ey = expand * h
 *   fx0 = (x - ex) * W, fx1 = ((x + w) + ex) * W, fy0 = (y - ey) * H, fy1 = ((y + h) + ey) * H      (W, H = frame_width, frame_height)
 *   a NaN among them drops the row; else each is clamped to [0, W] (resp. [0, H]), x0 = floor(fx0), x1 = ceil(fx1), y0 = floor(fy0),
 *   y1 = ceil(fy1), and the region is {n, r, x0, y0, x1 - x0, y1 - y0}.
 * The mapping is direct because run_frames / detect_frames stretch the whole frame to the model input (no letterbox). The first
 * `capacity` kept rows are written to rois_dev (snnb_roi[capacity]), entries past them are zeroed, and *count_dev = min(kept, capacity).
 * Checked on the host before anything is enqueued: non-null device or managed pointers of the context's device aligned to 4 bytes,
 * num_frames >= 1, 1 <= max_rows <= 100, frame size >= 1, capacity >= 1, expand finite and >= 0, a stream that is not capturing. */
int snnb_rois_from_detections(snnb_context* ctx, const float* rows_dev, const int* counts_dev, int num_frames, int max_rows, int frame_width,
                              int frame_height, const snnb_roi_select* sel, snnb_roi* rois_dev, int capacity, int* count_dev, void* stream);
/* Device-resident variant: inputs already uploaded with snnb_model_set_input(); forward only, asynchronous. */
int snnb_model_set_input(snnb_model* m, int idx, const float* host_input_nhwc);
int snnb_model_forward(snnb_model* m);
int snnb_model_get_output(snnb_model* m, int idx, float* host_output, size_t out_capacity);
/* Output of any layer (JSON index) as host NHWC fp32 — the per-layer checkpoint the reference's model tests compare
 * (demo/test/unittest/resnet18Test.cpp:85-198). Requires that the layer was not fused away (fuse=0) . */
int snnb_model_layer_output(snnb_model* m, int layer, float* host_nhwc, size_t capacity);
/* Dump every layer's output as "<dir>/<name> pass[0].dump" (vulkanBackend.cpp:108-143). */
int snnb_model_dump_outputs(snnb_model* m, const char* dir);
/* Per-layer device time of one forward pass, ms, via event pairs (writeTimeStat, core.cpp:437-442). times[num_layers]. */
int snnb_model_time_layers(snnb_model* m, float* times_ms, int capacity);
/* Name of the CUDA kernel layer `layer` launched in the last snnb_model_time_layers() pass ("" for a layer that launched none:
 * inputs, fused-away layers). What bench.py attributes the per-kernel roofline to. */
int snnb_model_layer_kernel(const snnb_model* m, int layer, char* name, int name_cap);
/* Kernels launched by one forward pass. */
int snnb_model_launches_per_forward(const snnb_model* m);
/* YOLO detection output of the last run (yololayer.cpp:177-226): rows {class, score, x, y, w, h}; returns the
 * number of boxes for image `n` via *count. */
int snnb_model_get_boxes(snnb_model* m, int n, float* rows6, int max_rows, int* count);
/* The packed weight arena (device pointer, bytes): rank 0 packs, the caller broadcasts it once with NCCL
 * (torch.distributed) and no collective ever runs on the forward path (SURVEY §8e). */
int snnb_model_weight_arena(snnb_model* m, void** device_ptr, size_t* bytes);

/* ---- multi-GPU: the ONE collective of the engine, in C++ (SURVEY §8b/e) --------------------------------------------
 * One process per GPU. Rank `root` packs the weights; every other rank receives the packed arena with a single ncclBroadcast
 * on the context's stream. NCCL is resolved at run time (the process's already-loaded libnccl.so.2 - e.g. PyTorch's - else
 * dlopen): the library has no link-time dependency on it. Bootstrap: rank 0 calls snnb_nccl_unique_id and ships the 128
 * bytes to the others by whatever means the host has (MPI, a file, torch.distributed), then every rank creates its
 * communicator. No collective ever runs on the forward path. (The reference is single-device: new surface, kept thin.) */
typedef struct snnb_comm snnb_comm;
int snnb_nccl_unique_id(unsigned char id128[128]);
int snnb_nccl_comm_create(snnb_context* ctx, int rank, int world_size, const unsigned char id128[128], snnb_comm** out);
int snnb_nccl_comm_destroy(snnb_comm* comm);
int snnb_bcast_weights(snnb_model* m, snnb_comm* comm, int root); /* asynchronous on the context's stream */

/* ---- layer registration: snn::dp::registerLayer(name, LayerCreator) (core/src/ic2/layerFactory.h:116-122) ------------
 * A host registers a creator for a layer `type` string; when a model file names that type, the creator is called with a
 * read-only view of the "Layer_<i>" JSON object (the accessors below = what ModelParser hands the reference's creators,
 * modelparser.h:60-157) and fills in the implementation: how the output dims follow from the inputs' and what to launch.
 * `run` works on the context's stream with this header's own operator launches (or its own kernels on the tensors' planes).
 * Registering an existing name replaces it, as registerLayer() does (built-in types included). */
typedef struct snnb_layer_json snnb_layer_json;
int snnb_layer_json_number(const snnb_layer_json* layer, const char* key, double* out);             /* 0 = present and numeric */
int snnb_layer_json_string(const snnb_layer_json* layer, const char* key, char* buf, int cap);      /* 0 = present and a string */
/* numeric array at a dotted path ("weights.kernel"); the pointer stays valid during the creator call only */
int snnb_layer_json_numbers(const snnb_layer_json* layer, const char* path, const double** data, size_t* count);
typedef struct {
    void* user;
    /* hwc triples: in_hwc[3*i .. 3*i+2] = (height, width, channels) of input i; write the output's into out_hwc[3]. 0 = ok. */
    int (*output_dims)(void* user, int num_inputs, const int* in_hwc, int* out_hwc);
    /* enqueue the layer's work on snnb_context_stream(ctx). 0 = ok. */
    int (*run)(void* user, snnb_context* ctx, int num_inputs, const snnb_tensor* const* inputs, snnb_tensor* output);
    void (*destroy)(void* user); /* may be NULL */
} snnb_layer_impl;
typedef int (*snnb_layer_creator)(void* registry_user, const snnb_layer_json* layer, snnb_layer_impl* out);
int snnb_register_layer(const char* type_name, snnb_layer_creator creator, void* registry_user);
int snnb_unregister_layer(const char* type_name);
/* Raw device planes of a tensor for custom kernels: NHWC, channel pitch `cp` (a multiple of 8), fp16 hi plane and lo plane
 * (value = hi + lo; lo is NULL in the half-precision storage mode). */
int snnb_tensor_planes(const snnb_tensor* t, void** hi, void** lo, int* cp);
/* Diagnostics: the work decomposition SNNB_ALGO_TCGEN05_STREAMK would use for `tiles` output tiles of `num_kb` K blocks on `sms` SMs,
 * evaluated on the host with the kernel's own arithmetic. rows = capacity x 6 ints {cta, tile, kb0, kb1, piece, pieces} in each CTA's
 * order; returns the number of rows (may exceed capacity), -1 when the tile count is a multiple of `sms` or too small to cut. No GPU needed. */
int snnb_debug_streamk_schedule(int tiles, int num_kb, int sms, int* rows, int capacity);
/* Diagnostics: the K layout of the stem kernel's feed mode for a k x k stride-`stride` convolution with `ic` input channels and x padding
 * `pad_x`: out = {px (left margin of the compact input copy), d (pixel offset of tap 0 in the window), nch (16-byte chunks per window),
 * ksteps (K = 16 steps per filter row), rows_per_panel (filter rows sharing one 128-byte weight row)}. Returns 1 if the layer can use
 * the feed mode, 0 if not. No GPU needed. */
int snnb_debug_feed_plan(int k, int stride, int pad_x, int ic, int out[5]);
/* Diagnostics: how a convolution would be run, decided on the host exactly as the engine and snnb_conv2d_launch decide it.
 * query = {in_h, in_w, in_c, out_h, out_w, out_c, k, stride, pad_x, pad_y, pad_mode, residual (0/1), algo (SNNB_ALGO_*),
 * may_prepad (0/1: a pre-padded copy of the input may be allocated), may_feed (0/1: the input is a model input that may carry the
 * compact feed copy), row_stride, row_pad (the weights' row-window operand; row_stride 0 = none), feed_pad (the weights' feed
 * operand; -1 = none)}. out = {path (0 refused, 1 CUDA cores, 2 implicit GEMM, 3 row window, 4 row window on the feed copy),
 * pad_x, pad_y, pad_mode (what the kernel sees), prepad_h, prepad_w (0 = no pre-padded copy), feed_h, feed_w, feed_py, feed_px
 * (0 = no feed copy)}. Returns 0. No GPU needed. */
int snnb_debug_conv_plan(const int query[18], int out[10]);
/* Diagnostics: the kernel instantiation of the most recent convolution launched on `ctx` (per-operator or inside a model's forward
 * pass): out = {path (as snnb_debug_conv_plan; 0 before any convolution), terms (product form of the tensor-core kernels: 3 fp32x3,
 * 2 fp16w, 1 fp16; 0 on the CUDA cores), n_blk (output channels per tile), ksplit (K pieces per tile, 1 = none), stream_k (0/1),
 * fks (K steps per filter row of the row-window kernel's feed mode, 0 otherwise)}. Host-side record, no GPU work. Returns 0. */
int snnb_debug_last_conv_variant(snnb_context* ctx, int out[6]);

#ifdef __cplusplus
}
#endif
#endif /* SNNB_H_ */
