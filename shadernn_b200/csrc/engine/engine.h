// Host engine of libsnn_b200.so — a from-scratch C++ counterpart of ShaderNN's model loading / graph building /
// execution stack, keeping its names so the mapping to the reference is one-to-one:
//
//   snn::dp::ModelParser            core/src/ic2/modelparser.{h,cpp}      JSON (+ sidecar .bin) model reader
//   snn::dp::<Op>Desc / <Op>Layer   core/src/ic2/<op>.{h,cpp}             per-op descs, dims, padding rules
//   snn::dp::registerLayer / createLayerInstance   layerFactory.{h,cpp}   string -> creator registry + aliases
//   snn::dp::loadFromJsonModel / generateInferenceGraph   dp.{h,cpp}      DAG wiring, Kahn toposort, dims
//   snn::MixedInferenceCore         core/inc/snn/core.h, core/src/ic2/core.cpp   stage list, init, run
//   snn::dp::CudaBackend            (new) backend.h's DeviceBackend role  streams, graphs, timers, dumps
//
// What differs by design: a batch dimension N, NHWC split-fp16 device tensors, weights BN-folded and packed once
// into a single device arena, one CUDA kernel launch per layer (fewer with fusion), optional CUDA-graph replay.
#pragma once

#include <algorithm>
#include <map>
#include <memory>
#include <string>
#include <vector>

#include "../snnb_internal.h"
#include "json.h"

namespace snn {

struct SNNModelOutputBoxes { // yololayer.cpp:219-225 rows {class, score, x, y, w, h}
    std::vector<std::vector<float>> rows;
};

namespace dp {

// -------------------------------------------------------------------------------------------------------------
// ModelParser (modelparser.h:30-157). Reads "numLayers", "Layer_<i>", optional "inputRange"; when
// numLayers.bin_file_name is present the weights stream from that sidecar file (raw LE fp32, layer order) which is
// looked up next to the JSON file.
// -------------------------------------------------------------------------------------------------------------
class ModelParser {
public:
    explicit ModelParser(const std::string& fileName);
    ~ModelParser();
    int getLayerCount() const;
    std::string getLayerName(int layerId) const; // "type", or "name" when type == "Lambda" (modelparser.cpp:78-86)
    int getNumInbound(int layerId) const;
    std::vector<int> getInboundLayerId(int layerId) const;
    int getInputPlanes(int layerId) const;
    int getOutputPlanes(int layerId) const;
    bool isInputRange01() const;
    const json::Value& layer(int layerId) const;
    bool isBinWeight() const { return binFile != nullptr; }
    // next `count` floats of the sidecar stream
    void readBin(float* dst, size_t count);
    const std::string& fileName() const { return _fileName; }

private:
    std::string _fileName;
    json::ValuePtr _root;
    FILE* binFile = nullptr;
};

// Padding spec as the parser leaves it: four strings, either all digits or a keyword ("same"/"valid"/"none")
// (modelparser.cpp:584-609), plus the conv "mode".
int padModeId(const std::string& mode); // SNNB_PAD_* of a padding mode string (conv2dVulkan.cpp:73-80)
struct PaddingSpec {
    std::string t = "valid", b = "valid", l = "valid", r = "valid";
    std::string mode; // "constant" | "replicate" | "reflect" | "" (unset)
    void parse(const json::Value& layerObj, bool readMode);
    // conv2d.cpp:39-74 / separableconvolution.cpp:27-62 / maxpool2d.cpp:37-72: {T, B, L, R}
    void offsets(int kernelSize, bool evenKernelTopLeftMinusOne, uint32_t (&offs)[4]) const;
    bool validLike() const { return t == "0" || t == "valid" || t == "none"; }
};

struct Dims {
    uint32_t width = 0, height = 0, depth = 0; // depth = channels here (the reference's IODesc carries both ceil(C/4) and C)
};

struct ActivationSpec {
    int id      = SNNB_ACT_NONE;
    float alpha = 0.0f;
    // Accepts every spelling the reference uses (SURVEY Q12): conv "leakyRelu", add/activation/dense "leaky_relu",
    // CPU map "SiLU"/"softmax"/"identity"/""; anything unknown is identity (conv2dVulkan.cpp:58-72).
    static int fromString(const std::string& s);
};

// -------------------------------------------------------------------------------------------------------------
// GenericModelLayer (genericlayer.h:60-139): graph node + execution unit.
// -------------------------------------------------------------------------------------------------------------
class GenericModelLayer {
public:
    virtual ~GenericModelLayer() {}
    std::string name;      // "<file> layer [NN] <Type>" (dp.cpp:135)
    std::string typeName;  // registry name after aliasing
    int layerId = -1;
    std::vector<GenericModelLayer*> prevLayers, nextLayers;
    std::vector<Dims> inputDims;
    uint32_t numInputPlanes = 0, numOutputPlanes = 0;
    bool isInputLayer = false;

    // genericlayer.cpp:64-90 default: out = uint32(scale*in + translate) per axis, depth = max input depth
    virtual void getOutputDims(uint32_t& width, uint32_t& height, uint32_t& depth) const;
    struct Transform { float scaleW = 1, scaleH = 1, transW = 0, transH = 0; };
    virtual Transform getOutputScaleDimAdjustment() const { return Transform(); }

    // ---- execution ----
    // fold/pack this layer's weights on the host (no device work); empty for weightless layers
    virtual void packWeights(snnb::PackedHost&) {}
    snnb_weights weights; // points into the model's arena after init
    std::vector<snnb_tensor*> inputs;
    snnb_tensor* output = nullptr;
    // GenericModelLayer::run -> RenderPass::run (genericlayer.cpp:39-62): enqueue this layer's kernel(s)
    virtual int run(snnb_context* ctx) = 0;
    // fusion bookkeeping (engine-level; see MixedInferenceCore::init)
    bool fusedAway          = false;      // produces nothing itself (its work happens inside another layer)
    snnb_tensor* residual   = nullptr;    // Conv2D: tensor added before the activation (fused Add)
    int fusedAct            = -1;         // Conv2D: activation taken over from a fused Add (-1 = own)
    float fusedAlpha        = 0.0f;
    float* scratch          = nullptr;    // per-layer device scratch (InstanceNorm stats)
    size_t scratchBytes() const { return _scratchBytes; }

protected:
    size_t _scratchBytes = 0;
};

// A layer supplied through the C-ABI (snnb_register_layer): dims and launches are the host's callbacks.
class PluginLayer : public GenericModelLayer {
public:
    snnb_layer_impl impl {};
    ~PluginLayer() override {
        if (impl.destroy) impl.destroy(impl.user);
    }
    void getOutputDims(uint32_t& w, uint32_t& h, uint32_t& d) const override;
    int run(snnb_context* ctx) override;
};

typedef GenericModelLayer* (*LayerCreator)(ModelParser&, int);
void initLayerRegisty();
void registerLayer(const std::string& layerName, LayerCreator creator);
GenericModelLayer* createLayerInstance(std::string layerName, ModelParser& parser, int i);

// -------------------------------------------------------------------------------------------------------------
// Layers
// -------------------------------------------------------------------------------------------------------------
struct InputLayerDesc {
    uint32_t inputWidth = 0, inputHeight = 0, inputChannels = 0, inputIndex = 0;
    void parse(ModelParser& parser, int layerId); // modelparser.cpp:480-497
};
class InputLayerLayer : public GenericModelLayer {
public:
    InputLayerDesc _desc;
    void getOutputDims(uint32_t& w, uint32_t& h, uint32_t& d) const override;
    int run(snnb_context*) override { return 0; }
};

struct GenericConvDesc {
    uint32_t kernelSize = 1, stride = 1;
    PaddingSpec padding;
    ActivationSpec activation;
    std::string activationName;
    std::vector<float> weights; // Conv2D: OIHW; depthwise: [C][k][k]
    std::vector<float> biases;  // empty when useBias is not "True"
    bool useBatchNormalization = false;
    std::map<std::string, std::vector<float>> batchNormalization; // gamma beta movingMean movingVariance
};
struct Conv2DDesc : GenericConvDesc {
    void parse(ModelParser& parser, int layerId); // modelparser.cpp:574-781
};
class Conv2DLayer : public GenericModelLayer {
public:
    Conv2DDesc _desc;
    // How this layer runs (made once at load by plan(); packWeights and run follow it). convPlan is the plan for the model's batch:
    // the core swaps in the plan made for each batch size (MixedInferenceCore::BatchPlan), with the path, padding and copies of this one.
    snnb::ConvQuery query;
    snnb::ConvPlan convPlan;
    // Replicate / reflect padding on the tensor path: the TMA unit can only zero-fill, so the engine materialises the
    // padded input (pad kernel, vk_pad.comp semantics) and runs the tensor-core kernel over it with zero padding.
    snnb_tensor* prepadded = nullptr;
    // Plans the layer once its input, output and residual tensors are known. mayFeed: the input is a model input that may carry
    // the compact 4-channel feed copy (snnb_tensor::feed_hi).
    void plan(int convAlgo, bool mayFeed, int precision, int smCount);
    Transform getOutputScaleDimAdjustment() const override; // conv2d.cpp:102-113
    void getOutputDims(uint32_t& w, uint32_t& h, uint32_t& d) const override;
    void packWeights(snnb::PackedHost& p) override;
    int run(snnb_context* ctx) override;
};
struct SeparableConv2DDesc : GenericConvDesc {
    void parse(ModelParser& parser, int layerId); // modelparser.cpp:783-985
};
class SeparableConv2DLayer : public GenericModelLayer { // depthwise (the name is historical)
public:
    SeparableConv2DDesc _desc;
    void getOutputDims(uint32_t& w, uint32_t& h, uint32_t& d) const override; // separableconvolution.cpp:77-86
    void packWeights(snnb::PackedHost& p) override;
    int run(snnb_context* ctx) override;
};
struct PoolDesc {
    uint32_t kernelSize = 1, stride = 1;
    PaddingSpec padding;
    void parseMax(ModelParser& parser, int layerId); // modelparser.cpp:304-371
    void parseAvg(ModelParser& parser, int layerId); // modelparser.cpp:373-397
};
class PoolingLayer : public GenericModelLayer { // MaxPooling2D / AveragePooling2D
public:
    PoolDesc _desc;
    bool isAvg = false;
    Transform getOutputScaleDimAdjustment() const override; // maxpool2d.cpp:26-35, avgpool2d.cpp:21-30
    int run(snnb_context* ctx) override;
};
class AdaptiveAvgPool2dLayer : public GenericModelLayer { // adaptiveavgpool2d.h (GL-only in the reference): pool -> pool x pool
public:
    uint32_t poolSize = 1;
    void getOutputDims(uint32_t& w, uint32_t& h, uint32_t& d) const override;
    int run(snnb_context* ctx) override;
};
class AddLayer : public GenericModelLayer { // addlayer.h:27-46
public:
    ActivationSpec activation;
    int run(snnb_context* ctx) override;
};
class BatchNormalizationLayer : public GenericModelLayer { // batchnorm.h:28-50
public:
    std::map<std::string, std::vector<float>> batchNormalization;
    ActivationSpec activation;
    void packWeights(snnb::PackedHost& p) override;
    int run(snnb_context* ctx) override;
};
class InstanceNormLayer : public GenericModelLayer { // instancenorm.h:28-54
public:
    std::vector<float> gamma, beta;
    ActivationSpec activation;
    void packWeights(snnb::PackedHost& p) override;
    int run(snnb_context* ctx) override;
    void setScratch() { _scratchBytes = 0; }
    void computeScratch(int n) { _scratchBytes = snnb::instnorm_scratch_floats(n, snnb::round_up((int) numOutputPlanes, 8)) * sizeof(float); }
};
class ActivationLayer : public GenericModelLayer { // activation.h:27-48 (creatable, not registered in the reference)
public:
    ActivationSpec activation;
    int run(snnb_context* ctx) override;
};
class DenseLayer : public GenericModelLayer { // denselayer.cpp:27-54
public:
    std::vector<float> kernel; // flat, [out][in]
    std::vector<float> biases;
    ActivationSpec activation;
    uint32_t units = 0;
    void getOutputDims(uint32_t& w, uint32_t& h, uint32_t& d) const override;
    void packWeights(snnb::PackedHost& p) override;
    int run(snnb_context* ctx) override;
    snnb_tensor* flat = nullptr; // staging when the input is not 1x1
    snnb::ConvQuery query;       // its 1x1 convolution, described at load by plan() once the tensors are known
    snnb::ConvPlan convPlan;     // ... and planned for the model's batch
    void plan(int precision, int smCount);
    GenericModelLayer* gapSource = nullptr; // fused head: global average pool of this layer's output feeds the Dense (core.cpp, fusion 4)
};
class FlattenLayer : public GenericModelLayer { // flattenlayer.cpp:29-62 (CPU flavour: HWC order)
public:
    ActivationSpec activation;
    void getOutputDims(uint32_t& w, uint32_t& h, uint32_t& d) const override;
    int run(snnb_context* ctx) override;
};
class ConcatenateLayer : public GenericModelLayer { // concatenation.h:25-40
public:
    void getOutputDims(uint32_t& w, uint32_t& h, uint32_t& d) const override;
    int run(snnb_context* ctx) override;
};
class UpSampling2DLayer : public GenericModelLayer { // upsampling2d.h:26-47
public:
    float scale = 1.0f;
    std::string interpolationType = "nearest";
    Transform getOutputScaleDimAdjustment() const override { return Transform {scale, scale, 0.0f, 0.0f}; }
    int run(snnb_context* ctx) override;
};
class PadLayer : public GenericModelLayer { // padlayer.{h,cpp}
public:
    PaddingSpec padding;
    std::string mode = "constant"; // the reference parser never overwrites it (modelparser.cpp:1112-1113 drops the argument)
    Transform getOutputScaleDimAdjustment() const override; // padlayer.cpp:60-68
    int run(snnb_context* ctx) override;
};
class SubpixelLayer : public GenericModelLayer { // subpixelmerge.h:26-47
public:
    uint32_t kernelSize = 2;
    void getOutputDims(uint32_t& w, uint32_t& h, uint32_t& d) const override;
    int run(snnb_context* ctx) override;
};
class YOLOLayer : public GenericModelLayer { // yololayer.{h,cpp}: host decode + NMS of two heads
public:
    void getOutputDims(uint32_t& w, uint32_t& h, uint32_t& d) const override;
    int run(snnb_context*) override { return 0; } // executed by the core after the device pass (candidates + host NMS)
    // all-host decode (downloads both heads): the fallback when an image has more candidates than the device list holds
    int decode(snnb_context* ctx, std::vector<SNNModelOutputBoxes>& perImage);
    // device threshold + compaction into `devCounts` / `devCand` ([N] ints, [N][YOLO_MAX_CAND][8] floats), asynchronous
    // one slot per (image, cell, anchor) of both heads: the list can never overflow, whatever the scores. Layout: 32-byte header
    // (word 0 = number of candidates) + rows of 8 floats. The host copies the header and the first YOLO_HEAD_ROWS rows with every
    // submission; the (rare) rest is fetched in wait().
    static constexpr int YOLO_HEAD_ROWS = 2048;
    // sizes for `n` images: buffers are allocated for the loaded batch and used for the model's batch
    int maxCand(int n) const { return inputs.size() < 2 ? 0 : n * (inputs[0]->h * inputs[0]->w + inputs[1]->h * inputs[1]->w) * 3; }
    size_t candidateBytes(int n) const { return 32 + (size_t) maxCand(n) * 8 * sizeof(float); }
    size_t headBytes(int n) const { return 32 + (size_t) std::min(maxCand(n), YOLO_HEAD_ROWS) * 8 * sizeof(float); }
    int enqueueCandidates(snnb_context* ctx, void* devBuf);
    // host part on the downloaded buffer of `n` images: exact score formula, confidence threshold, score sort, NMS (yololayer.cpp:56-164).
    // Returns 0, or -1 when some image overflowed the candidate list (caller falls back to decode()).
    int finishDecode(const void* hostBuf, const void* devBuf, int n, std::vector<SNNModelOutputBoxes>& perImage) const;
};

// -------------------------------------------------------------------------------------------------------------
// dp.h: model loading + graph generation
// -------------------------------------------------------------------------------------------------------------
struct ShaderGenOptions { // layeroption.h:27-48, trimmed to what a CUDA backend can honour, + batch
    uint32_t desiredInputWidth = 0, desiredInputHeight = 0; // desiredInput[0] (dp.cpp:505-507)
    uint32_t batch             = 1;
    int convAlgo               = SNNB_ALGO_AUTO;
    bool fuse                  = false;
    bool useCudaGraph          = false;
    int precision              = SNNB_PRECISION_FP32X3; // layeroption.h:43 preferrHalfPrecision <-> SNNB_PRECISION_FP16
};

std::vector<std::shared_ptr<GenericModelLayer>> loadFromJsonModel(const std::string& fileName); // dp.cpp:115-167
// Kahn topological sort over nextLayers (dp.cpp:389-429), dims propagation (dp.cpp:432-640).
struct InferenceGraph {
    std::vector<GenericModelLayer*> sorted; // execution order, inputs first
    std::vector<Dims> outputDims;           // per sorted layer
};
InferenceGraph generateInferenceGraph(const std::vector<std::shared_ptr<GenericModelLayer>>& layers, const ShaderGenOptions& options);

} // namespace dp

// -------------------------------------------------------------------------------------------------------------
// MixedInferenceCore (core.h:66-146, core.cpp): owns the stages' tensors, the weight arena, the CUDA graph.
// -------------------------------------------------------------------------------------------------------------
class MixedInferenceCore {
public:
    ~MixedInferenceCore();
    static std::unique_ptr<MixedInferenceCore> create(snnb_context* ctx, const std::string& modelFileName, const dp::ShaderGenOptions& options,
                                                      std::string& err);
    // forward pass only (inputs already resident in the InputLayers' tensors); asynchronous
    int forward();
    // host -> input tensor idx (async H2D + split kernel)
    int setInput(int idx, const float* hostNHWC);
    // output idx -> host NHWC (merge kernel + D2H, synchronous)
    int getOutput(int idx, float* host, size_t capacityFloats);
    // run(RunParameters) end to end (core.cpp:97-245): H2D, forward, D2H, class index
    int run(const float* hostInput, float* hostOutput, size_t capacityFloats, int* classes1);
    // streaming: double-buffered submit/wait (H2D of batch i+1 overlaps compute of batch i)
    int submit(const float* hostInput, float* hostOutput, size_t capacityFloats, int* classes1, int* ticket);
    // same with a u8 NHWC image batch, normalised on the device as (x - mean[c]) * norm[c] (imageTexture.h:114)
    int submitU8(const uint8_t* hostInput, const float mean[4], const float norm[4], float* hostOutput, size_t capacityFloats, int* classes1, int* ticket);
    int submitImpl(const void* hostInput, bool u8, const float* mean, const float* norm, float* hostOutput, size_t capacityFloats, int* classes1, int* ticket,
                   const snnb_image_io* io = nullptr);
    int submitImage(const snnb_image_io& io, int* ticket);
    int wait(int ticket);
    // snnb_model_run_device: device buffers in and out, fenced against the caller's stream (NULL: the context's); asynchronous
    int runDevice(const snnb_device_buffer* inputs, int numInputs, const snnb_device_buffer* outputs, int numOutputs, int* classes1Dev, cudaStream_t stream);
    // snnb_model_detect_device: runDevice's inputs and fences, then YOLO decode + score sort + NMS on the device into rows / counts
    int detectDevice(const snnb_device_buffer* inputs, int numInputs, float* rowsDev, int maxRows, int* countsDev, cudaStream_t stream);
    // snnb_model_run_frames / snnb_model_detect_frames: runDevice / detectDevice with device video frames as input 0
    int runFrames(const snnb_frames* frames, const snnb_device_buffer* outputs, int numOutputs, int* classes1Dev, cudaStream_t stream);
    int detectFrames(const snnb_frames* frames, float* rowsDev, int maxRows, int* countsDev, cudaStream_t stream);
    // snnb_model_transform_frames: runFrames' input and fences, then output 0 written as device video frames
    int transformFrames(const snnb_frames* frames, const snnb_frames_out* out, cudaStream_t stream);
    // snnb_model_transform_luma: the frames' Y plane into a 1-channel model, output 0 (1 channel) out as the Y plane, chroma resampled
    int transformLuma(const snnb_frames* frames, const snnb_frames_out* out, cudaStream_t stream);
    // snnb_model_segment_frames: runFrames' input (luma: transformLuma's), output 0's scores resampled and reduced to an 8-bit label plane
    int segmentFrames(const snnb_frames* frames, bool luma, const snnb_labels_out* out, cudaStream_t stream);
    // snnb_model_run_rois: runFrames with regions of numFrames frames as the batch; slots without a valid region come out zero
    int runRois(const snnb_frames* frames, int numFrames, const snnb_roi* roisDev, const int* countDev, const snnb_device_buffer* outputs, int numOutputs,
                int* classes1Dev, cudaStream_t stream);
    // snnb_model_run_frame_list / detect_frame_list / run_rois_list: runFrames / detectFrames / runRois with one descriptor per image
    int runFrameList(const snnb_frame_list* frames, const snnb_device_buffer* outputs, int numOutputs, int* classes1Dev, cudaStream_t stream);
    int detectFrameList(const snnb_frame_list* frames, float* rowsDev, int maxRows, int* countsDev, cudaStream_t stream);
    int runRoisList(const snnb_frame_list* frames, const snnb_roi* roisDev, const int* countDev, const snnb_device_buffer* outputs, int numOutputs,
                    int* classes1Dev, cudaStream_t stream);
    // snnb_model_detect_rois / detect_rois_list: runRois' input and forward pass, the device decode per slot, then the slots' rows mapped
    // to their frames and merged by one NMS per frame
    int detectRois(const snnb_frames* frames, int numFrames, const snnb_roi* roisDev, const int* countDev, float* rowsDev, int maxRows, int* countsDev,
                   cudaStream_t stream);
    int detectRoisList(const snnb_frame_list* frames, const snnb_roi* roisDev, const int* countDev, float* rowsDev, int maxRows, int* countsDev,
                       cudaStream_t stream);
    // snnb_model_transform_frame_list / transform_luma_list / segment_frame_list: transformFrames / transformLuma / segmentFrames with a
    // frame list in and one output descriptor per image out
    int transformFrameList(const snnb_frame_list* frames, const snnb_frame_out_list* out, cudaStream_t stream);
    int transformLumaList(const snnb_frame_list* frames, const snnb_frame_out_list* out, cudaStream_t stream);
    int segmentFrameList(const snnb_frame_list* frames, bool luma, const snnb_labels_list* out, cudaStream_t stream);
    int layerOutput(int layerId, float* host, size_t capacityFloats);
    int timeLayers(std::vector<float>& ms);
    int dumpOutputs(const std::string& dir);
    // snnb_model_set_batch: every later call works on n images, 1 <= n <= options.batch, in the first n images of the loaded batch's
    // storage. Host-side: plans n on its first use, switches to it on every later one; nothing is enqueued or allocated.
    int setBatch(int n);
    int batch() const { return curBatch; } // the model's batch: images per call (options.batch is the capacity)
    // snnb_model_set_count_batches: the sizes a region call with a device-side count runs its forward pass at (count_body). Host-side:
    // plans each size as setBatch does and drops every dispatch graph already built; a refused call changes nothing.
    int setCountBatches(const int* sizes, int numSizes);

    snnb_context* ctx = nullptr;
    dp::ShaderGenOptions options;
    std::vector<std::shared_ptr<dp::GenericModelLayer>> layers; // JSON order
    dp::InferenceGraph graph;
    std::vector<dp::GenericModelLayer*> inputLayers, outputLayers;
    std::vector<SNNModelOutputBoxes> boxes; // per image, when the model ends in a YOLO layer
    void* arena       = nullptr;
    size_t arenaBytes = 0;
    int launchesPerForward = 0; // of the model's batch (0 until its first forward pass has counted them)
    bool isClassifier = false;
    std::vector<std::string> layerKernels; // per layer (JSON order): the kernel its last timeLayers() pass launched

private:
    bool init(std::string& err);
    int enqueueForward(bool countOnly);
    std::vector<snnb_tensor*> ownedTensors;
    void* scratchArena = nullptr;
    // What one batch size runs with: a ConvPlan per layer of `planned` (Conv2D and Dense, in that order), made by the planner for n
    // images, and (use_cuda_graph) the forward pass captured at n after one eager pass has counted its launches and grown the split-K
    // scratch. Made on first use and kept for the model's life; storage is the loaded batch's for every n.
    struct BatchPlan {
        std::vector<snnb::ConvPlan> plans;
        int launches = 0; // kernels of one forward pass (0: not counted yet)
        cudaGraph_t graph = nullptr;
        cudaGraphExec_t exec = nullptr;
        // The dispatch graph of a region call with a device-side count at this batch (setCountBatches): the selector node, then a chain
        // of IF nodes, one per body of `bodies`, each holding the forward pass at its size. Built on the first such call at this batch.
        cudaGraph_t dispatch = nullptr;
        cudaGraphExec_t dispatchExec = nullptr;
        cudaGraphNode_t selector = nullptr;
        snnb::CountBodies bodies;
        void dropDispatch() {
            if (dispatchExec) cudaGraphExecDestroy(dispatchExec);
            if (dispatch) cudaGraphDestroy(dispatch);
            dispatch = nullptr, dispatchExec = nullptr, selector = nullptr;
        }
    };
    std::map<int, BatchPlan> batchPlans;
    std::vector<dp::GenericModelLayer*> planned;
    int curBatch = 0;
    BatchPlan* cur = nullptr;
    std::vector<int> countSizes; // setCountBatches' sizes (empty: a device-side count does not size the forward pass)
    std::string makeBatchPlan(int n, BatchPlan& b) const; // "" or why the plans at n cannot run on the loaded batch's storage
    void useBatch(int n, const BatchPlan& b);             // makes b's plans (made for n images) and n-image tensor extents current
    int captureForward(BatchPlan& b);
    int buildDispatch(const char* api, const int* countDev); // the current batch's dispatch graph (host-synchronous)
    int forwardCounted(const int* countDev);                 // the forward pass at count_body's size of *countDev; asynchronous
    float* ioStage   = nullptr; // device fp32 staging for input/output conversion (stable address: graph-safe)
    size_t ioStageBytes = 0;
    int* argmaxDev   = nullptr;
    dp::YOLOLayer* yolo = nullptr;
    void* yoloDev  = nullptr; // device candidate lists of the YOLO decode (counts + [N][YOLO_MAX_CAND][8])
    void* yoloHost = nullptr; // pinned host mirror
    int decodeYolo(void* dev, void* host, bool sync); // candidates kernel + D2H (+ sync + host NMS into `boxes`)
    // streaming state
    static constexpr size_t SMALL_RESULT_BYTES = 64 * 1024;
    struct Slot {
        void* stageResize = nullptr; // device staging of a differently-sized u8 input (grown on demand)
        size_t stageResizeBytes = 0;
        float* stageIn = nullptr;   // device fp32 staging for this slot's input batch
        float* stageOut = nullptr;  // device fp32 staging for output 0
        int* argmax = nullptr;
        cudaEvent_t h2dDone = nullptr, stageFree = nullptr, resultReady = nullptr;
        int* classesHost = nullptr;
        // small classifier results bypass the copy engine: one kernel writes values + arg-max into this mapped pinned block, wait() hands
        // them to the caller's buffers (two ~10 us device->host copy commands less per batch)
        void* smallHost = nullptr;      // cudaHostAlloc'ed, SMALL_RESULT_BYTES
        void* smallDev  = nullptr;      // its device alias
        float* userOut = nullptr;       // where wait() copies the values
        int* userClasses = nullptr;     // ... and the 1-based classes
        size_t userFloats = 0;
        void* yoloDev = nullptr;
        void* yoloHost = nullptr;
        int n = 0; // the model's batch when this slot's submission was made: what wait() delivers
        bool busy = false, everUsed = false;
    } slots[2];
    cudaStream_t copyStream = nullptr;
    int nextTicket = 0;
    int ensureStreaming();
    // runDevice's fences: the caller's stream -> the context's stream (callerReady), and back (deviceDone); created on first use
    cudaEvent_t callerReady = nullptr, deviceDone = nullptr;
    // What a device-resident call feeds the model: one snnb_device_buffer per input, or (frames != NULL) a batch of frames into input 0,
    // or (rois != NULL as well) regions of numFrames frames, one per batch slot, with roiCount (NULL: all slots) of them used, or
    // (luma) the frames' Y plane alone into a 1-channel input, or (list != NULL, in place of frames) a frame list: one descriptor per
    // image, the model's batch of them, or with rois its list->count (= numFrames) source frames.
    // The input staging (and, for regions, the clearing of the slots without one) is the only step in which these entry points differ.
    struct DeviceFeed {
        const snnb_device_buffer* inputs = nullptr;
        int numInputs = 0;
        const snnb_frames* frames = nullptr;
        const snnb_frame_list* list = nullptr;
        const snnb_roi* rois = nullptr;
        const int* roiCount = nullptr;
        int numFrames = 0;
        bool luma = false;
    };
    // shared by runDevice, detectDevice, runFrames, detectFrames, runRois and their frame-list forms: the host-side checks of the feed and the stream (nothing
    // enqueued), then the fenced input staging + forward pass, the outputs or the detections, and the fence back to the caller's stream
    int runDeviceFeed(const char* api, const DeviceFeed& in, const snnb_device_buffer* outputs, int numOutputs, int* classes1Dev, cudaStream_t stream);
    int detectDeviceFeed(const char* api, const DeviceFeed& in, float* rowsDev, int maxRows, int* countsDev, cudaStream_t stream);
    int detectRoisFeed(const char* api, const DeviceFeed& in, float* rowsDev, int maxRows, int* countsDev, cudaStream_t stream);
    // shared by the frame-writing calls and their list forms: the feed's checks, then out's (one batch description `o`, or the output
    // list `ol`), output 0's, the forward pass, the output kernel and the fence
    int transformDeviceFeed(const char* api, const DeviceFeed& in, const snnb_frames_out* o, const snnb_frame_out_list* ol, cudaStream_t stream);
    int transformLumaDeviceFeed(const char* api, const DeviceFeed& in, const snnb_frames_out* o, const snnb_frame_out_list* ol, cudaStream_t stream);
    int segmentDeviceFeed(const char* api, const DeviceFeed& in, const snnb_labels_out* o, const snnb_labels_list* ol, cudaStream_t stream);
    int checkDeviceFeed(const char* api, const DeviceFeed& in, cudaStream_t stream);
    // regions with a device-side count, once sizes are declared: the forward pass is the dispatch graph's (forwardCounted)
    bool counted(const DeviceFeed& in) const { return in.rois && in.roiCount && !countSizes.empty(); }
    int prepareCounted(const char* api, const DeviceFeed& in); // a counted call's capture check and dispatch graph (host-side, before any enqueue)
    // detectDeviceFeed's and detectRoisFeed's host checks of max_rows, the feed, rows, counts and the heads, and the decode's scratch
    int checkDetectOutputs(const char* api, const DeviceFeed& in, float* rowsDev, int maxRows, int* countsDev, cudaStream_t stream);
    int enqueueDeviceForward(const DeviceFeed& in, cudaStream_t stream);
    int fenceToCaller(cudaStream_t stream);
    void* detectScratch = nullptr; // detectDevice's per-image keys (yolo_detect_scratch_bytes), allocated on first use
    // detectRois' scratch, sized for the loaded batch: the per-slot rows [B][100][6] and counts [B], the merge's two row buffers
    // (roi_merge_scratch_bytes), then one {start, length} per frame for roiSegsCap frames; allocated on first use, and again for a call
    // with more frames than roiSegsCap
    void* roiScratch = nullptr;
    int roiSegsCap   = 0;
};

} // namespace snn
