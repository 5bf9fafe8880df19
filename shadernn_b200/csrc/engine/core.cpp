// MixedInferenceCore: init (tensor plan, weight arena, fusion, CUDA-graph capture) and run.
// Counterpart of core/src/ic2/core.cpp:294-410 (init) and :97-245 (run).
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <type_traits>
#include <unordered_map>
#include <unordered_set>

#include "engine.h"

using namespace snnb;

namespace snn {

using namespace dp;

MixedInferenceCore::~MixedInferenceCore() {
    if (ctx) {
        cudaSetDevice(ctx->device);
        cudaStreamSynchronize(ctx->stream);
    }
    for (auto& kv : batchPlans) {
        if (kv.second.exec) cudaGraphExecDestroy(kv.second.exec);
        if (kv.second.graph) cudaGraphDestroy(kv.second.graph);
        kv.second.dropDispatch();
    }
    for (auto* t : ownedTensors) snnb_tensor_free(t);
    if (arena) cudaFree(arena);
    if (scratchArena) cudaFree(scratchArena);
    if (ioStage) cudaFree(ioStage);
    if (argmaxDev) cudaFree(argmaxDev);
    if (yoloDev) cudaFree(yoloDev);
    if (yoloHost) cudaFreeHost(yoloHost);
    for (auto& sl : slots) {
        if (sl.yoloDev) cudaFree(sl.yoloDev);
        if (sl.yoloHost) cudaFreeHost(sl.yoloHost);
        if (sl.stageIn) cudaFree(sl.stageIn);
        if (sl.stageResize) cudaFree(sl.stageResize);
        if (sl.stageOut) cudaFree(sl.stageOut);
        if (sl.smallHost) cudaFreeHost(sl.smallHost);
        if (sl.argmax) cudaFree(sl.argmax);
        if (sl.h2dDone) cudaEventDestroy(sl.h2dDone);
        if (sl.stageFree) cudaEventDestroy(sl.stageFree);
        if (sl.resultReady) cudaEventDestroy(sl.resultReady);
    }
    if (copyStream) cudaStreamDestroy(copyStream);
    if (callerReady) cudaEventDestroy(callerReady);
    if (detectScratch) cudaFree(detectScratch);
    if (roiScratch) cudaFree(roiScratch);
    if (deviceDone) cudaEventDestroy(deviceDone);
}

std::unique_ptr<MixedInferenceCore> MixedInferenceCore::create(snnb_context* ctx, const std::string& modelFileName, const ShaderGenOptions& options,
                                                               std::string& err) {
    std::unique_ptr<MixedInferenceCore> core(new MixedInferenceCore());
    core->ctx     = ctx;
    core->options = options;
    try {
        core->layers = loadFromJsonModel(modelFileName);
        core->graph  = generateInferenceGraph(core->layers, options);
    } catch (std::exception& e) {
        err = e.what();
        return nullptr;
    }
    if (!core->init(err)) return nullptr;
    return core;
}

static bool allZeroPadding(const PaddingSpec& p) {
    uint32_t o[4];
    p.offsets(3, true, o); // kernel size only matters for "same"
    const bool keyword_same = !(p.t == "valid" || p.t == "none" || (!p.t.empty() && std::all_of(p.t.begin(), p.t.end(), ::isdigit)));
    return !keyword_same && o[0] == 0 && o[1] == 0 && o[2] == 0 && o[3] == 0;
}

bool MixedInferenceCore::init(std::string& err) {
    const int N = (int) options.batch;
    // ShaderGenOptions::preferrHalfPrecision (layeroption.h:43 -> RGBA16F textures): every tensor is ONE fp16 plane
    const bool twoPlanes = options.precision != SNNB_PRECISION_FP16;
    std::unordered_map<GenericModelLayer*, int> order;
    for (size_t i = 0; i < graph.sorted.size(); ++i) order[graph.sorted[i]] = (int) i;

    for (auto* L : graph.sorted) {
        if (L->isInputLayer) inputLayers.push_back(L);
        if (L->nextLayers.empty()) outputLayers.push_back(L);
        if (L->typeName == "YOLO") yolo = static_cast<YOLOLayer*>(L);
    }
    std::stable_sort(inputLayers.begin(), inputLayers.end(), [](GenericModelLayer* a, GenericModelLayer* b) {
        return static_cast<InputLayerLayer*>(a)->_desc.inputIndex < static_cast<InputLayerLayer*>(b)->_desc.inputIndex;
    });
    if (inputLayers.empty()) {
        err = "model has no InputLayer";
        return false;
    }

    // ---- fusion passes (engine-level; off => one kernel per reference layer, every layer output observable) ----
    // `alias[L]` = the layer whose output tensor stands in for L's (L launches nothing).
    std::unordered_map<GenericModelLayer*, GenericModelLayer*> alias;
    if (options.fuse) {
        for (auto* L : graph.sorted) {
            // (1) Pad -> Conv2D/Depthwise with zero own padding: the consumer's gather applies the offsets (and mode) itself.
            if (L->typeName == "Pad" && L->nextLayers.size() == 1 && L->prevLayers.size() == 1) {
                auto* pad  = static_cast<PadLayer*>(L);
                auto* next = L->nextLayers[0];
                PaddingSpec* np = nullptr;
                if (next->typeName == "Conv2D" && static_cast<Conv2DLayer*>(next)->_desc.kernelSize > 1) np = &static_cast<Conv2DLayer*>(next)->_desc.padding;
                if (next->typeName == "SeparableConv2D" && pad->mode == "constant") np = &static_cast<SeparableConv2DLayer*>(next)->_desc.padding;
                if (np && allZeroPadding(*np)) {
                    uint32_t o[4];
                    pad->padding.offsets(0, false, o);
                    np->t = std::to_string(o[0]), np->b = std::to_string(o[1]), np->l = std::to_string(o[2]), np->r = std::to_string(o[3]);
                    np->mode       = pad->mode;
                    L->fusedAway   = true;
                    alias[L]       = L->prevLayers[0];
                }
            }
            // (2) Conv2D(linear) -> Add(+act): the conv's epilogue adds the other operand and applies the Add's activation.
            if (L->typeName == "Add" && L->prevLayers.size() == 2) {
                auto* add = static_cast<AddLayer*>(L);
                GenericModelLayer* a = L->prevLayers[0];
                GenericModelLayer* b = L->prevLayers[1];
                auto fusable = [&](GenericModelLayer* c, GenericModelLayer* other) {
                    if (c->typeName != "Conv2D" || c->nextLayers.size() != 1 || c->fusedAway) return false;
                    auto* conv = static_cast<Conv2DLayer*>(c);
                    if (conv->_desc.activation.id != SNNB_ACT_NONE || conv->residual || conv->fusedAct >= 0) return false;
                    return order[other] < order[c] && c != other; // the other operand must be complete before the conv runs
                };
                GenericModelLayer* conv = nullptr;
                GenericModelLayer* other = nullptr;
                if (fusable(b, a))
                    conv = b, other = a;
                else if (fusable(a, b))
                    conv = a, other = b;
                if (conv) {
                    conv->fusedAct   = add->activation.id;
                    conv->fusedAlpha = add->activation.alpha;
                    conv->prevLayers.push_back(other); // bookkeeping only: residual operand
                    L->fusedAway     = true;           // the Add launches nothing; its tensor is written by the conv
                    alias[conv]      = L;              // conv output == add output
                }
            }
            // (4) global AveragePooling2D -> [Flatten] -> Dense with few units: one classifier-head launch (gap_dense_kernel).
            if (L->typeName == "Dense" && L->prevLayers.size() == 1) {
                GenericModelLayer* f = L->prevLayers[0];
                GenericModelLayer* pool = (f->typeName == "Flatten" && f->prevLayers.size() == 1 && f->nextLayers.size() == 1 &&
                                           static_cast<FlattenLayer*>(f)->activation.id == SNNB_ACT_NONE)
                                              ? f->prevLayers[0]
                                              : f;
                auto dimsOf = [&](GenericModelLayer* x) { return graph.outputDims[order[x]]; };
                if (pool->typeName == "AveragePooling2D" && static_cast<PoolingLayer*>(pool)->isAvg && pool->nextLayers.size() == 1 && pool->prevLayers.size() == 1 &&
                    !pool->fusedAway && dimsOf(pool).width * dimsOf(pool).height == 1 && static_cast<DenseLayer*>(L)->units <= 256 &&
                    dimsOf(pool->prevLayers[0]).width * dimsOf(pool->prevLayers[0]).height >= 4 && dimsOf(pool->prevLayers[0]).depth <= 4096 &&
                    // a head that does not fit the kernel's shared memory runs as pool + Dense: the pool must then write its tensor
                    gap_dense_parts((int) dimsOf(pool->prevLayers[0]).depth, (int) static_cast<DenseLayer*>(L)->units) > 0 &&
                    static_cast<PoolingLayer*>(pool)->_desc.kernelSize >= dimsOf(pool->prevLayers[0]).width &&
                    static_cast<PoolingLayer*>(pool)->_desc.kernelSize >= dimsOf(pool->prevLayers[0]).height) {
                    static_cast<DenseLayer*>(L)->gapSource = pool->prevLayers[0];
                    pool->fusedAway = true; // launches nothing; keeps its own (unwritten) 1x1 tensor so that shapes downstream still check
                }
            }
            // (3) Flatten of a 1x1xC tensor without activation is the identity.
            if (L->typeName == "Flatten" && L->inputDims.size() == 1 && L->inputDims[0].width * L->inputDims[0].height == 1 &&
                static_cast<FlattenLayer*>(L)->activation.id == SNNB_ACT_NONE) {
                L->fusedAway = true;
                alias[L]     = L->prevLayers[0];
            }
        }
    }

    // ---- tensors: one output per executing layer (core.cpp:356-374 allocates one texture per stage) ----
    std::unordered_map<GenericModelLayer*, snnb_tensor*> outOf;
    auto resolve = [&](GenericModelLayer* L) -> GenericModelLayer* {
        std::unordered_set<GenericModelLayer*> seen;
        while (alias.count(L) && !seen.count(L)) {
            seen.insert(L);
            L = alias[L];
        }
        return L;
    };
    for (size_t i = 0; i < graph.sorted.size(); ++i) {
        GenericModelLayer* L = graph.sorted[i];
        if (L->typeName == "YOLO") continue; // host op
        GenericModelLayer* owner = resolve(L);
        if (owner != L && !(L->typeName == "Conv2D")) continue; // Pad/Flatten aliases own nothing
        if (outOf.count(owner)) continue;
        // dims of the tensor = dims of `owner` (for conv->add fusion both agree)
        const Dims& d = graph.outputDims[order[owner]];
        snnb_tensor* t = nullptr;
        if (tensor_alloc(ctx, N, (int) d.height, (int) d.width, (int) d.depth, &t, twoPlanes)) {
            err = get_error();
            return false;
        }
        ownedTensors.push_back(t);
        outOf[owner] = t;
    }
    for (auto* L : graph.sorted) {
        if (L->typeName == "YOLO") {
            for (auto* p : L->prevLayers) L->inputs.push_back(outOf.at(resolve(p)));
            continue;
        }
        GenericModelLayer* owner = resolve(L);
        L->output                = outOf.count(owner) ? outOf[owner] : nullptr;
        if (L->fusedAway) continue;
        size_t nin = L->prevLayers.size();
        if (L->typeName == "Conv2D" && static_cast<Conv2DLayer*>(L)->fusedAct >= 0) {
            nin -= 1; // last prev is the residual operand
            L->residual = outOf.at(resolve(L->prevLayers.back()));
        }
        for (size_t k = 0; k < nin; ++k) L->inputs.push_back(outOf.at(resolve(L->prevLayers[k])));
        if (L->typeName == "Conv2D") {
            auto* cl = static_cast<Conv2DLayer*>(L);
            static const bool noFeed = getenv("SNNB_NO_FEED") != nullptr;
            snnb_tensor* in          = L->inputs[0];
            cl->plan(options.convAlgo, !noFeed && resolve(L->prevLayers[0])->isInputLayer && !in->feed_hi, options.precision,
                     ctx->sm_count); // the first stem reading an input gets its feed
            planned.push_back(L);
            const ConvPlan& p = cl->convPlan;
            if (p.prepad_h) {
                if (tensor_alloc(ctx, N, p.prepad_h, p.prepad_w, in->c, &cl->prepadded, twoPlanes)) {
                    err = get_error();
                    return false;
                }
                ownedTensors.push_back(cl->prepadded);
            }
            if (p.path == CONV_ROWWIN_FEED && tensor_alloc_feed(in, p.feed_h, p.feed_w, p.feed_py, p.feed_px)) {
                err = get_error();
                return false;
            }
        }
        if (L->typeName == "Dense") {
            auto* dl = static_cast<DenseLayer*>(L);
            if (L->inputs[0]->h * L->inputs[0]->w != 1) {
                if (tensor_alloc(ctx, N, 1, 1, (int) dl->numInputPlanes, &dl->flat, twoPlanes)) {
                    err = get_error();
                    return false;
                }
                ownedTensors.push_back(dl->flat);
            }
            if ((uint32_t) (L->inputs[0]->h * L->inputs[0]->w * L->inputs[0]->c) != dl->numInputPlanes) {
                err = L->name + ": Dense expects " + std::to_string(dl->numInputPlanes) + " inputs, graph provides " +
                      std::to_string(L->inputs[0]->h * L->inputs[0]->w * L->inputs[0]->c);
                return false;
            }
            dl->plan(options.precision, ctx->sm_count);
            planned.push_back(L);
        }
        if ((L->typeName == "Add" || L->typeName == "Concatenate") && L->inputs.size() != 2) {
            err = L->name + ": expects exactly two inputs";
            return false;
        }
        // The kernels index weights and operands with the RUNTIME tensors' extents: a model whose declared planes disagree with
        // what the graph produces would read out of bounds on the device. Reject it here, as a load error.
        auto dimsStr = [](const snnb_tensor* t) { return std::to_string(t->h) + "x" + std::to_string(t->w) + "x" + std::to_string(t->c); };
        if (L->typeName == "Conv2D" || L->typeName == "SeparableConv2D" || L->typeName == "BatchNormalization" || L->typeName == "InstanceNorm") {
            if (L->inputs.empty() || !L->output) {
                err = L->name + ": layer has no input";
                return false;
            }
            if ((uint32_t) L->inputs[0]->c != L->numInputPlanes) {
                err = L->name + ": inputPlanes " + std::to_string(L->numInputPlanes) + " but the producing layer has " + std::to_string(L->inputs[0]->c) + " channels";
                return false;
            }
            const uint32_t wantOut = (L->typeName == "Conv2D") ? L->numOutputPlanes : L->numInputPlanes;
            if ((uint32_t) L->output->c != wantOut) {
                err = L->name + ": output tensor has " + std::to_string(L->output->c) + " channels, weights are packed for " + std::to_string(wantOut);
                return false;
            }
        }
        if (L->typeName == "Add") {
            for (auto* in : L->inputs)
                if (in->h != L->output->h || in->w != L->output->w || in->c != L->output->c) {
                    err = L->name + ": Add operand " + dimsStr(in) + " does not match the output " + dimsStr(L->output);
                    return false;
                }
        }
        if (L->typeName == "Conv2D" && L->residual &&
            (L->residual->h != L->output->h || L->residual->w != L->output->w || L->residual->c != L->output->c)) {
            err = L->name + ": fused Add operand " + dimsStr(L->residual) + " does not match the output " + dimsStr(L->output);
            return false;
        }
        if (L->typeName == "Concatenate") {
            if (L->inputs[0]->h != L->inputs[1]->h || L->inputs[0]->w != L->inputs[1]->w || L->inputs[0]->c + L->inputs[1]->c != L->output->c ||
                L->inputs[0]->h != L->output->h || L->inputs[0]->w != L->output->w) {
                err = L->name + ": Concatenate operands " + dimsStr(L->inputs[0]) + " and " + dimsStr(L->inputs[1]) + " do not stack into " + dimsStr(L->output);
                return false;
            }
        }
    }

    // input tensors whose ONLY readers are feed-mode stems need no regular planes (snnb_tensor::feed_only)
    for (auto* in : inputLayers) {
        snnb_tensor* t = in->output;
        if (!t || !t->feed_hi || getenv("SNNB_NO_FEED_ONLY")) continue;
        bool only = true;
        int readers = 0;
        for (auto* L : graph.sorted) {
            if (L->fusedAway || L->isInputLayer) continue;
            const bool reads = std::find(L->inputs.begin(), L->inputs.end(), t) != L->inputs.end() || L->residual == t;
            if (!reads) continue;
            ++readers;
            only = only && L->typeName == "Conv2D" && static_cast<Conv2DLayer*>(L)->convPlan.path == CONV_ROWWIN_FEED && L->inputs.size() >= 1 && L->inputs[0] == t && L->residual != t &&
                   std::count(L->inputs.begin(), L->inputs.end(), t) == 1;
        }
        for (auto* o : outputLayers) only = only && o->output != t; // a model that returns its input
        t->feed_only = only && readers > 0;
    }

    // ---- weights: fold + pack on the host, then ONE device arena (broadcastable with a single NCCL call) ----
    std::vector<std::pair<GenericModelLayer*, PackedHost>> packed;
    size_t total = 0, scratchTotal = 0;
    for (auto* L : graph.sorted) {
        PackedHost p;
        try {
            L->packWeights(p);
        } catch (std::exception& e) {
            err = L->name + ": " + e.what();
            return false;
        }
        if (p.kind) {
            total += p.device_bytes();
            packed.emplace_back(L, std::move(p));
        }
        if (L->typeName == "InstanceNorm") {
            static_cast<InstanceNormLayer*>(L)->computeScratch(N);
            scratchTotal += (L->scratchBytes() + 255) & ~(size_t) 255;
        }
    }
    arenaBytes = total ? total : 256;
    if (cudaMalloc(&arena, arenaBytes) != cudaSuccess) {
        err = "cudaMalloc(weight arena) failed";
        return false;
    }
    {
        char* cur = (char*) arena;
        for (auto& pr : packed) {
            if (place_weights(ctx, pr.second, cur, &pr.first->weights)) {
                err = get_error();
                return false;
            }
            cur += pr.first->weights.bytes;
        }
    }
    if (scratchTotal) {
        if (cudaMalloc(&scratchArena, scratchTotal) != cudaSuccess) {
            err = "cudaMalloc(scratch) failed";
            return false;
        }
        char* cur = (char*) scratchArena;
        for (auto* L : graph.sorted)
            if (L->scratchBytes()) {
                L->scratch = (float*) cur;
                cur += (L->scratchBytes() + 255) & ~(size_t) 255;
            }
    }

    // ---- io staging (stable addresses so the captured graph stays valid) ----
    size_t maxFloats = 1;
    for (auto* L : inputLayers) maxFloats = std::max(maxFloats, L->output->pixels() * (size_t) L->output->c);
    for (auto* L : outputLayers)
        if (L->output) maxFloats = std::max(maxFloats, L->output->pixels() * (size_t) L->output->c);
    ioStageBytes = maxFloats * sizeof(float);
    if (cudaMalloc(&ioStage, ioStageBytes) != cudaSuccess || cudaMalloc(&argmaxDev, sizeof(int) * N) != cudaSuccess) {
        err = "cudaMalloc(io staging) failed";
        return false;
    }
    if (yolo) {
        const size_t yb = yolo->candidateBytes(N);
        if (cudaMalloc(&yoloDev, yb) != cudaSuccess || cudaMallocHost(&yoloHost, yb) != cudaSuccess) {
            err = "cudaMalloc(YOLO candidate lists) failed";
            return false;
        }
    }
    {
        GenericModelLayer* last = nullptr;
        for (auto* L : outputLayers)
            if (L->output) {
                last = L;
                break;
            }
        isClassifier = last && last->output->h == 1 && last->output->w == 1 && last->output->c > 1;
    }

    // ---- the loaded batch is the model's first batch: its plans are the ones made above ----
    curBatch = N;
    cur      = &batchPlans[N];
    for (auto* L : planned) cur->plans.push_back(L->typeName == "Conv2D" ? static_cast<Conv2DLayer*>(L)->convPlan : static_cast<DenseLayer*>(L)->convPlan);

    // ---- one eager pass: counts launches and warms everything up; then optionally capture ----
    const uint64_t before = ctx->launches;
    if (enqueueForward(false)) {
        err = get_error();
        return false;
    }
    cur->launches = launchesPerForward = (int) (ctx->launches - before);
    if (cudaStreamSynchronize(ctx->stream) != cudaSuccess) {
        err = std::string("first forward pass failed: ") + cudaGetErrorString(cudaGetLastError());
        return false;
    }
    if (options.useCudaGraph && captureForward(*cur)) {
        err = get_error();
        return false;
    }
    return true;
}

// The forward pass at the model's batch captured into b's graph. Run after an eager pass at that batch: that pass made every lazily
// allocated resource (tensor-map encoder, split-K scratch), and neither cudaMalloc nor a synchronous memset may run in a capture.
int MixedInferenceCore::captureForward(BatchPlan& b) {
    const uint64_t keep = ctx->launches;
    SNNB_CUDA_OK(cudaStreamBeginCapture(ctx->stream, cudaStreamCaptureModeThreadLocal));
    const int rc        = enqueueForward(false);
    const cudaError_t e = cudaStreamEndCapture(ctx->stream, &b.graph);
    ctx->launches       = keep;
    if (rc) return rc;
    SNNB_CUDA_OK(e);
    SNNB_CUDA_OK(cudaGraphInstantiate(&b.exec, b.graph, 0));
    return 0;
}

// Each Conv2D and Dense layer planned for n images by the same planner and query as at load. The kernel, the pre-padded copy and the
// feed copy were allocated and packed for the load-time plan, so they must come out the same at every n; a planner whose path choice
// depended on n would otherwise read a copy that was never allocated.
std::string MixedInferenceCore::makeBatchPlan(int n, BatchPlan& b) const {
    b.plans.clear();
    for (size_t i = 0; i < planned.size(); ++i) {
        GenericModelLayer* L = planned[i];
        const bool conv      = L->typeName == "Conv2D";
        ConvQuery q          = conv ? static_cast<Conv2DLayer*>(L)->query : static_cast<DenseLayer*>(L)->query;
        q.n                  = n;
        const ConvPlan p     = plan_conv(q);
        const ConvPlan& at   = batchPlans.at((int) options.batch).plans[i];
        if (p.path != at.path || p.pad_x != at.pad_x || p.pad_y != at.pad_y || p.pad_mode != at.pad_mode || p.prepad_h != at.prepad_h ||
            p.prepad_w != at.prepad_w || p.feed_h != at.feed_h || p.feed_w != at.feed_w || p.feed_py != at.feed_py || p.feed_px != at.feed_px)
            return L->name + ": the plan for " + std::to_string(n) + " images (path " + std::to_string(p.path) + ", pre-padded " +
                   std::to_string(p.prepad_h) + " x " + std::to_string(p.prepad_w) + ", feed " + std::to_string(p.feed_h) + " x " +
                   std::to_string(p.feed_w) + ") differs from the loaded batch's (path " + std::to_string(at.path) + ", pre-padded " +
                   std::to_string(at.prepad_h) + " x " + std::to_string(at.prepad_w) + ", feed " + std::to_string(at.feed_h) + " x " +
                   std::to_string(at.feed_w) + ") beyond its launch configuration";
        b.plans.push_back(p);
    }
    return std::string();
}

int MixedInferenceCore::setBatch(int n) {
    SNNB_REQUIRE(n >= 1 && n <= (int) options.batch, "snnb_model_set_batch: batch %d; the model was loaded for 1 to %u images", n, options.batch);
    auto it = batchPlans.find(n);
    if (it == batchPlans.end()) {
        BatchPlan b;
        const std::string why = makeBatchPlan(n, b);
        SNNB_REQUIRE(why.empty(), "snnb_model_set_batch: %s", why.c_str());
        it = batchPlans.emplace(n, std::move(b)).first;
    }
    cur = &it->second, curBatch = n, launchesPerForward = cur->launches;
    useBatch(n, *cur);
    return 0;
}

void MixedInferenceCore::useBatch(int n, const BatchPlan& b) {
    for (size_t i = 0; i < planned.size(); ++i) {
        GenericModelLayer* L = planned[i];
        (L->typeName == "Conv2D" ? static_cast<Conv2DLayer*>(L)->convPlan : static_cast<DenseLayer*>(L)->convPlan) = b.plans[i];
    }
    for (auto* t : ownedTensors) t->n = n; // NHWC, image outermost: the first n images of every tensor are a prefix of its storage
}

int MixedInferenceCore::setCountBatches(const int* sizes, int numSizes) {
    const char* api = "snnb_model_set_count_batches";
    SNNB_REQUIRE(numSizes >= 0 && numSizes <= COUNT_BATCHES_MAX, "%s: %d sizes; 0 to %d may be declared", api, numSizes, COUNT_BATCHES_MAX);
    SNNB_REQUIRE(sizes || numSizes == 0, "%s: null sizes", api);
    SNNB_REQUIRE(options.useCudaGraph, "%s: the model was loaded without use_cuda_graph; the forward pass is chosen by the count inside a CUDA graph", api);
    for (int i = 0; i < numSizes; ++i)
        SNNB_REQUIRE(sizes[i] >= 1 && sizes[i] <= (int) options.batch && (i == 0 || sizes[i] > sizes[i - 1]),
                     "%s: sizes[%d] = %d; sizes must be strictly increasing, from 1 to the loaded batch of %u", api, i, sizes[i], options.batch);
    std::map<int, BatchPlan> made; // every size planned before anything changes
    for (int i = 0; i < numSizes; ++i) {
        if (batchPlans.count(sizes[i])) continue;
        BatchPlan b;
        const std::string why = makeBatchPlan(sizes[i], b);
        SNNB_REQUIRE(why.empty(), "%s: size %d: %s", api, sizes[i], why.c_str());
        made.emplace(sizes[i], std::move(b));
    }
    bool built = false;
    for (auto& kv : batchPlans) built = built || kv.second.dispatchExec;
    if (built) SNNB_CUDA_OK(cudaStreamSynchronize(ctx->stream)); // no dispatch graph is destroyed while a launch of it may be in flight
    for (auto& kv : batchPlans) kv.second.dropDispatch();
    for (auto& kv : made) batchPlans.emplace(kv.first, std::move(kv.second));
    countSizes.assign(sizes, sizes + numSizes);
    return 0;
}

// The dispatch graph of the model's batch B, built on the first counted region call at B, host-synchronously and before anything of that
// call is enqueued. Bodies: each declared size below B, then B. For each, one eager pass at that size if none ran yet (it counts the
// launches and grows the split-K scratch, which a capture cannot), then its forward pass captured into the body of an IF node. The
// IF nodes hang in a chain after the selector; each has its own handle, reset to 0 at every launch, and the selector sets one of them.
int MixedInferenceCore::buildDispatch(const char* api, const int* countDev) {
    BatchPlan& top = *cur;
    const int B    = curBatch;
    CountBodies b;
    for (int s : countSizes)
        if (s < B) b.size[b.num++] = s;
    b.size[b.num++] = B;
    cudaGraph_t g = nullptr;
    SNNB_CUDA_OK(cudaGraphCreate(&g, 0));
    cudaGraphNode_t selector = nullptr;
    const int rc = [&]() -> int {
        for (int k = 0; k < b.num; ++k) {
            const cudaError_t e = cudaGraphConditionalHandleCreate(&b.handle[k], g, 0, cudaGraphCondAssignDefault);
            SNNB_REQUIRE(e == cudaSuccess, "%s: cudaGraphConditionalHandleCreate: %s", api, cudaGetErrorString(e));
        }
        if (count_select_add(g, &selector, countDev, b)) return 1;
        cudaGraphNode_t prev = selector;
        for (int k = 0; k < b.num; ++k) {
            BatchPlan& p = batchPlans.at(b.size[k]);
            useBatch(b.size[k], p);
            if (!p.launches) {
                const uint64_t before = ctx->launches;
                if (int r = enqueueForward(false)) return r;
                p.launches = (int) (ctx->launches - before);
            }
            cudaGraphNodeParams cp = {};
            cp.type               = cudaGraphNodeTypeConditional;
            cp.conditional.handle = b.handle[k];
            cp.conditional.type   = cudaGraphCondTypeIf;
            cp.conditional.size   = 1;
            cudaGraphNode_t node  = nullptr;
            SNNB_CUDA_OK(cudaGraphAddNode(&node, g, &prev, 1, &cp));
            const uint64_t keep = ctx->launches;
            SNNB_CUDA_OK(cudaStreamBeginCaptureToGraph(ctx->stream, cp.conditional.phGraph_out[0], nullptr, nullptr, 0, cudaStreamCaptureModeThreadLocal));
            const int r = enqueueForward(false);
            cudaGraph_t body    = nullptr;
            const cudaError_t e = cudaStreamEndCapture(ctx->stream, &body);
            ctx->launches       = keep;
            if (r) return r;
            SNNB_CUDA_OK(e);
            prev = node;
        }
        return 0;
    }();
    useBatch(B, top);
    launchesPerForward = top.launches;
    cudaGraphExec_t exec = nullptr;
    cudaError_t e        = rc ? cudaSuccess : cudaStreamSynchronize(ctx->stream); // the eager passes
    cudaGraphInstantiateParams ip = {};
    if (!rc && e == cudaSuccess) e = cudaGraphInstantiateWithParams(&exec, g, &ip);
    if (rc || e != cudaSuccess) {
        cudaGraphDestroy(g);
        if (!rc) set_error("%s: the dispatch graph at batch %d: %s (instantiation result %d)", api, B, cudaGetErrorString(e), (int) ip.result_out);
        return rc ? rc : 1;
    }
    top.dispatch = g, top.dispatchExec = exec, top.selector = selector, top.bodies = b;
    return 0;
}

int MixedInferenceCore::forwardCounted(const int* countDev) {
    if (count_select_set(cur->dispatchExec, cur->selector, countDev, cur->bodies)) return 1;
    SNNB_CUDA_OK(cudaGraphLaunch(cur->dispatchExec, ctx->stream));
    ctx->launches += 1 + (uint64_t) cur->launches; // the selector and, as an upper bound, the forward pass at the model's batch
    return 0;
}

int MixedInferenceCore::enqueueForward(bool) {
    // SNNB_SYNC_LAYERS: debugging aid - wait for every layer and name the one whose kernel faulted (eager passes only)
    static const bool syncLayers = getenv("SNNB_SYNC_LAYERS") != nullptr;
    cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
    if (syncLayers) cudaStreamIsCapturing(ctx->stream, &cap);
    const bool capturing = cap != cudaStreamCaptureStatusNone;
    for (auto* L : graph.sorted) {
        if (L->fusedAway || L->isInputLayer || L->typeName == "YOLO") continue;
        if (int rc = L->run(ctx)) return rc;
        if (syncLayers && !capturing) {
            const cudaError_t e = cudaStreamSynchronize(ctx->stream);
            if (e != cudaSuccess) {
                set_error("%s (%s): %s", L->name.c_str(), ctx->last_kernel ? ctx->last_kernel : "?", cudaGetErrorString(e));
                return 1;
            }
        }
    }
    return 0;
}

int MixedInferenceCore::forward() {
    if (cur->exec) {
        SNNB_CUDA_OK(cudaGraphLaunch(cur->exec, ctx->stream));
        ctx->launches += (uint64_t) cur->launches;
        return 0;
    }
    // the first forward pass at a batch size (every pass without use_cuda_graph) runs eagerly and counts its launches; with
    // use_cuda_graph it is init's warm-up pass for that size, and the graph is captured right after it (unless the context's stream is
    // itself being captured, by snnb_graph_capture_begin: that capture records this pass)
    const uint64_t before = ctx->launches;
    if (int rc = enqueueForward(false)) return rc;
    cur->launches = launchesPerForward = (int) (ctx->launches - before);
    if (options.useCudaGraph) {
        cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
        SNNB_CUDA_OK(cudaStreamIsCapturing(ctx->stream, &cap));
        if (cap == cudaStreamCaptureStatusNone) return captureForward(*cur);
    }
    return 0;
}

int MixedInferenceCore::setInput(int idx, const float* host) {
    SNNB_REQUIRE(idx >= 0 && idx < (int) inputLayers.size() && host, "setInput: bad argument");
    snnb_tensor* t     = inputLayers[idx]->output;
    const size_t bytes = t->pixels() * t->c * sizeof(float);
    SNNB_CUDA_OK(cudaMemcpyAsync(ioStage, host, bytes, cudaMemcpyHostToDevice, ctx->stream));
    return launch_split_f32(ctx, ioStage, t);
}

int MixedInferenceCore::getOutput(int idx, float* host, size_t capacityFloats) {
    SNNB_REQUIRE(idx >= 0 && idx < (int) outputLayers.size() && host, "getOutput: bad argument");
    GenericModelLayer* L = outputLayers[idx];
    if (L->typeName == "YOLO") { // rows of image 0 .. N-1 are fetched with snnb_model_get_boxes
        set_error("getOutput: output %d is a YOLO detection list; use snnb_model_get_boxes", idx);
        return 2;
    }
    snnb_tensor* t      = L->output;
    const size_t floats = t->pixels() * t->c;
    SNNB_REQUIRE(capacityFloats >= floats, "getOutput: buffer too small (%zu < %zu floats)", capacityFloats, floats);
    if (launch_merge_f32(ctx, t, ioStage)) return 1;
    SNNB_CUDA_OK(cudaMemcpyAsync(host, ioStage, floats * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
    SNNB_CUDA_OK(cudaStreamSynchronize(ctx->stream));
    return 0;
}

int MixedInferenceCore::run(const float* hostInput, float* hostOutput, size_t capacityFloats, int* classes1) {
    if (setInput(0, hostInput)) return 1;
    if (forward()) return 1;
    if (yolo && decodeYolo(yoloDev, yoloHost, true)) return 1;
    int outIdx = -1;
    for (size_t i = 0; i < outputLayers.size(); ++i)
        if (outputLayers[i]->typeName != "YOLO") {
            outIdx = (int) i;
            break;
        }
    if (classes1 && isClassifier && outIdx >= 0) {
        if (launch_argmax(ctx, outputLayers[outIdx]->output, argmaxDev)) return 1;
        SNNB_CUDA_OK(cudaMemcpyAsync(classes1, argmaxDev, sizeof(int) * curBatch, cudaMemcpyDeviceToHost, ctx->stream));
    }
    if (hostOutput && outIdx >= 0) {
        if (getOutput(outIdx, hostOutput, capacityFloats)) return 1;
    } else {
        SNNB_CUDA_OK(cudaStreamSynchronize(ctx->stream));
    }
    if (classes1 && isClassifier && outIdx >= 0)
        for (int i = 0; i < curBatch; ++i) classes1[i] += 1; // core.cpp:228-233: argmax + 1
    return 0;
}

// YOLO decode: threshold + compaction on the device (yololayer.cpp:115-164 up to the confidence test), a few KB of candidates
// to the host, then the exact score formula, score sort and NMS there (identical lists, identical order: finishDecode).
int MixedInferenceCore::decodeYolo(void* dev, void* host, bool sync) {
    if (yolo->enqueueCandidates(ctx, dev)) return 1;
    SNNB_CUDA_OK(cudaMemcpyAsync(host, dev, yolo->headBytes(curBatch), cudaMemcpyDeviceToHost, ctx->stream)); // count + the first rows
    if (!sync) return 0;
    SNNB_CUDA_OK(cudaStreamSynchronize(ctx->stream));
    const int rc = yolo->finishDecode(host, dev, curBatch, boxes);
    if (rc < 0) return yolo->decode(ctx, boxes); // an image overflowed its candidate list: all-host decode of the (still resident) heads
    return rc;
}

// ---- streaming (additive to the reference's synchronous run) ---------------------------------------------------------
int MixedInferenceCore::ensureStreaming() {
    if (copyStream) return 0;
    SNNB_CUDA_OK(cudaStreamCreateWithFlags(&copyStream, cudaStreamNonBlocking));
    for (auto& sl : slots) {
        SNNB_CUDA_OK(cudaMalloc(&sl.stageIn, ioStageBytes));
        SNNB_CUDA_OK(cudaMalloc(&sl.stageOut, ioStageBytes));
        SNNB_CUDA_OK(cudaMalloc(&sl.argmax, sizeof(int) * options.batch));
        SNNB_CUDA_OK(cudaHostAlloc(&sl.smallHost, SMALL_RESULT_BYTES, cudaHostAllocMapped));
        SNNB_CUDA_OK(cudaHostGetDevicePointer(&sl.smallDev, sl.smallHost, 0));
        SNNB_CUDA_OK(cudaEventCreateWithFlags(&sl.h2dDone, cudaEventDisableTiming));
        SNNB_CUDA_OK(cudaEventCreateWithFlags(&sl.stageFree, cudaEventDisableTiming));
        SNNB_CUDA_OK(cudaEventCreateWithFlags(&sl.resultReady, cudaEventDisableTiming));
        if (yolo) {
            SNNB_CUDA_OK(cudaMalloc(&sl.yoloDev, yolo->candidateBytes((int) options.batch)));
            SNNB_CUDA_OK(cudaMallocHost(&sl.yoloHost, yolo->candidateBytes((int) options.batch)));
        }
    }
    return 0;
}

int MixedInferenceCore::submit(const float* hostInput, float* hostOutput, size_t capacityFloats, int* classes1, int* ticket) {
    return submitImpl(hostInput, false, nullptr, nullptr, hostOutput, capacityFloats, classes1, ticket);
}
int MixedInferenceCore::submitU8(const uint8_t* hostInput, const float mean[4], const float norm[4], float* hostOutput, size_t capacityFloats, int* classes1, int* ticket) {
    SNNB_REQUIRE(mean && norm, "submitU8: null mean / norm");
    return submitImpl(hostInput, true, mean, norm, hostOutput, capacityFloats, classes1, ticket);
}
int MixedInferenceCore::submitImage(const snnb_image_io& io, int* ticket) {
    SNNB_REQUIRE(io.input_u8 && io.src_height > 0 && io.src_width > 0, "submit_image: bad input");
    SNNB_REQUIRE(!(io.output_f32 && io.output_u8), "submit_image: choose ONE of output_f32 / output_u8");
    return submitImpl(io.input_u8, true, io.mean4, io.norm4, io.output_f32, io.output_capacity, io.classes_1based, ticket, &io);
}
int MixedInferenceCore::submitImpl(const void* hostInput, bool u8, const float* mean, const float* norm, float* hostOutput, size_t capacityFloats, int* classes1,
                                   int* ticket, const snnb_image_io* io) {
    SNNB_REQUIRE(hostInput && ticket, "submit: null argument");
    if (ensureStreaming()) return 1;
    Slot& sl = slots[nextTicket & 1];
    SNNB_REQUIRE(!sl.busy, "submit: two submissions are already in flight; wait() on ticket %d first", nextTicket - 2);
    int outIdx = 0;
    snnb_tensor* in  = inputLayers[0]->output;
    snnb_tensor* out = outputLayers[outIdx]->output; // nullptr for a detection model: its output is the box list (snnb_model_get_boxes)
    if (!out) hostOutput = nullptr, classes1 = nullptr;
    const bool resize = io && (io->src_height != in->h || io->src_width != in->w);
    const size_t inBytes = resize ? (size_t) in->n * io->src_height * io->src_width * in->c : in->pixels() * in->c * (u8 ? sizeof(uint8_t) : sizeof(float));
    const size_t outFloats = out ? out->pixels() * out->c : 0;
    SNNB_REQUIRE(!hostOutput || capacityFloats >= outFloats, "submit: output buffer too small (%zu < %zu floats)", capacityFloats, outFloats);
    SNNB_REQUIRE(!(io && io->output_u8) || (out && io->output_capacity >= outFloats), "submit_image: u8 output buffer too small or the model has no tensor output");
    void* stage = sl.stageIn;
    if (resize) { // a source image of another size does not fit the model-sized staging: its own buffer, grown on demand
        if (inBytes > sl.stageResizeBytes) {
            SNNB_CUDA_OK(cudaStreamSynchronize(ctx->stream));
            if (sl.stageResize) SNNB_CUDA_OK(cudaFree(sl.stageResize));
            SNNB_CUDA_OK(cudaMalloc(&sl.stageResize, inBytes));
            sl.stageResizeBytes = inBytes;
        }
        stage = sl.stageResize;
    }
    // copy stream: wait until the split kernel of the submission that last used this slot has consumed the staging
    if (sl.everUsed) SNNB_CUDA_OK(cudaStreamWaitEvent(copyStream, sl.stageFree, 0));
    SNNB_CUDA_OK(cudaMemcpyAsync(stage, hostInput, inBytes, cudaMemcpyHostToDevice, copyStream));
    SNNB_CUDA_OK(cudaEventRecord(sl.h2dDone, copyStream));
    // compute stream
    SNNB_CUDA_OK(cudaStreamWaitEvent(ctx->stream, sl.h2dDone, 0));
    if (resize) {
        if (launch_resize_u8(ctx, reinterpret_cast<const uint8_t*>(stage), io->src_height, io->src_width, in, mean, norm, io->linear_filter != 0)) return 1;
    } else if (u8 ? launch_split_u8(ctx, reinterpret_cast<const uint8_t*>(sl.stageIn), in, mean, norm) : launch_split_f32(ctx, sl.stageIn, in)) {
        return 1;
    }
    SNNB_CUDA_OK(cudaEventRecord(sl.stageFree, ctx->stream));
    if (forward()) return 1;
    sl.userOut = nullptr, sl.userClasses = nullptr, sl.userFloats = 0;
    // a small classifier result (values + classes) is written straight into mapped pinned memory by ONE kernel; wait() copies it out
    static const bool noSmall = getenv("SNNB_NO_SMALL_RESULT") != nullptr;
    const bool small = !noSmall && isClassifier && !(io && io->output_u8) && (hostOutput || classes1) &&
                       outFloats * sizeof(float) + curBatch * sizeof(int) <= SMALL_RESULT_BYTES;
    if (small) {
        float* vals = static_cast<float*>(sl.smallDev);
        int* cls    = reinterpret_cast<int*>(static_cast<char*>(sl.smallDev) + outFloats * sizeof(float));
        if (launch_result_small(ctx, out, hostOutput ? vals : nullptr, classes1 ? cls : nullptr)) return 1;
        sl.userOut = hostOutput, sl.userClasses = classes1, sl.userFloats = outFloats;
        hostOutput = nullptr, classes1 = nullptr; // served
    }
    if (hostOutput) {
        if (launch_merge_f32(ctx, out, sl.stageOut)) return 1;
        SNNB_CUDA_OK(cudaMemcpyAsync(hostOutput, sl.stageOut, outFloats * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
    }
    if (io && io->output_u8) { // the output as an 8-bit image: clamp(round(v * scale + offset), 0, 255) on the device, a quarter of the bytes back
        if (launch_merge_u8(ctx, out, reinterpret_cast<uint8_t*>(sl.stageOut), io->out_scale, io->out_offset)) return 1;
        SNNB_CUDA_OK(cudaMemcpyAsync(io->output_u8, sl.stageOut, outFloats, cudaMemcpyDeviceToHost, ctx->stream));
    }
    sl.classesHost = nullptr;
    if (classes1 && isClassifier) {
        if (launch_argmax(ctx, out, sl.argmax)) return 1;
        SNNB_CUDA_OK(cudaMemcpyAsync(classes1, sl.argmax, sizeof(int) * curBatch, cudaMemcpyDeviceToHost, ctx->stream));
        sl.classesHost = classes1;
    }
    if (yolo && decodeYolo(sl.yoloDev, sl.yoloHost, false)) return 1; // candidates -> pinned host, asynchronously; NMS in wait()
    SNNB_CUDA_OK(cudaEventRecord(sl.resultReady, ctx->stream));
    sl.n    = curBatch;
    sl.busy = sl.everUsed = true;
    *ticket = nextTicket++;
    return 0;
}

int MixedInferenceCore::wait(int ticket) {
    SNNB_REQUIRE(ticket >= 0 && ticket < nextTicket && ticket >= nextTicket - 2, "wait: ticket %d is not in flight", ticket);
    Slot& sl = slots[ticket & 1];
    SNNB_REQUIRE(sl.busy, "wait: ticket %d was already waited for", ticket);
    SNNB_CUDA_OK(cudaEventSynchronize(sl.resultReady));
    if (sl.userOut) std::memcpy(sl.userOut, sl.smallHost, sl.userFloats * sizeof(float));
    if (sl.userClasses) {
        const int* cls = reinterpret_cast<const int*>(static_cast<const char*>(sl.smallHost) + sl.userFloats * sizeof(float));
        for (int i = 0; i < sl.n; ++i) sl.userClasses[i] = cls[i] + 1; // core.cpp:228-233: argmax + 1
    }
    sl.userOut = nullptr, sl.userClasses = nullptr;
    if (sl.classesHost)
        for (int i = 0; i < sl.n; ++i) sl.classesHost[i] += 1; // core.cpp:228-233: argmax + 1
    sl.busy = false;
    if (yolo) {
        const int rc = yolo->finishDecode(sl.yoloHost, sl.yoloDev, sl.n, boxes);
        SNNB_REQUIRE(rc >= 0, "wait: corrupt detection candidate list");
        return rc;
    }
    return 0;
}

// ---- device-resident inputs and outputs on the caller's stream (snnb_model_run_device) -------------------------------------
static const char* memoryTypeName(cudaMemoryType t) {
    switch (t) {
    case cudaMemoryTypeUnregistered: return "unregistered host memory";
    case cudaMemoryTypeHost: return "pinned host memory";
    case cudaMemoryTypeDevice: return "device memory";
    case cudaMemoryTypeManaged: return "managed memory";
    }
    return "unknown memory";
}
// A pointer the kernels may dereference: device or managed memory of `device`, aligned to its `elem`-byte elements.
static int checkDevicePointer(const char* api, const void* p, size_t elem, int device, const char* what, int idx) {
    SNNB_REQUIRE(p, "%s: %s %d: null data pointer", api, what, idx);
    cudaPointerAttributes a {};
    const cudaError_t e = cudaPointerGetAttributes(&a, p);
    if (e != cudaSuccess) cudaGetLastError(); // not sticky: leave no error behind for the next call
    SNNB_REQUIRE(e == cudaSuccess, "%s: %s %d: cudaPointerGetAttributes(%p) failed: %s", api, what, idx, p, cudaGetErrorString(e));
    SNNB_REQUIRE((a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged) && a.device == device,
                 "%s: %s %d: %p is %s of device %d; device or managed memory of device %d is required", api, what, idx, p, memoryTypeName(a.type), a.device,
                 device);
    SNNB_REQUIRE(reinterpret_cast<uintptr_t>(p) % elem == 0, "%s: %s %d: %p is not aligned to its %zu-byte elements", api, what, idx, p, elem);
    return 0;
}
static int checkDeviceBuffer(const char* api, const snnb_device_buffer& b, int device, const char* what, int idx) {
    SNNB_REQUIRE(b.dtype == SNNB_DTYPE_F32 || b.dtype == SNNB_DTYPE_F16 || b.dtype == SNNB_DTYPE_U8, "%s: %s %d: unknown dtype %d", api, what, idx, b.dtype);
    SNNB_REQUIRE(b.layout == SNNB_LAYOUT_NHWC || b.layout == SNNB_LAYOUT_NCHW, "%s: %s %d: unknown layout %d", api, what, idx, b.layout);
    const size_t elem = b.dtype == SNNB_DTYPE_F32 ? 4 : (b.dtype == SNNB_DTYPE_F16 ? 2 : 1);
    return checkDevicePointer(api, b.data, elem, device, what, idx);
}

// The row bytes of plane p of `width`-pixel frames (NV12 / NV21 rows of ceil(w/2) UV pairs, I420 rows of ceil(w/2) samples, P010 the
// NV12 rows in 16-bit samples), 0 for an unused plane.
static long long frameRowBytes(int format, int width, int p) {
    const long long cw = (width + 1) / 2;
    switch (format) {
    case SNNB_FRAME_NV12:
    case SNNB_FRAME_NV21: return p == 0 ? width : (p == 1 ? 2 * cw : 0);
    case SNNB_FRAME_I420: return p == 0 ? width : cw;
    case SNNB_FRAME_RGBA8: return p == 0 ? 4LL * width : 0;
    case SNNB_FRAME_P010: return p == 0 ? 2LL * width : (p == 1 ? 4 * cw : 0);
    }
    return 0;
}
static bool knownFrameFormat(int format) { return (format >= SNNB_FRAME_NV12 && format <= SNNB_FRAME_RGBA8) || format == SNNB_FRAME_P010; }

// Image i of frames in either form, as an snnb_frames: a batch (snnb_frames, snnb_frames_out) is one description whose images lie at its
// image strides, so it is image i for every i; a list image is a one-image description at stride 0. Only input frames have a matrix.
template <class Batch, class List>
static snnb_frames frameImage(const Batch* b, const List* l, int i) {
    snnb_frames m {};
    if (b) {
        m.format = b->format, m.width = b->width, m.height = b->height;
        for (int p = 0; p < 3; ++p) m.plane[p] = b->plane[p], m.pitch[p] = b->pitch[p], m.image_stride[p] = b->image_stride[p];
    } else {
        m.format = l->format, m.width = l->images[i].width, m.height = l->images[i].height;
        for (int p = 0; p < 3; ++p) m.plane[p] = l->images[i].plane[p], m.pitch[p] = l->images[i].pitch[p];
    }
    if constexpr (std::is_same<Batch, snnb_frames>::value) m.matrix = b ? b->matrix : l->images[i].matrix;
    return m;
}
static snnb_labels_image labelsImage(const snnb_labels_out* o, const snnb_labels_list* ol, int i) {
    if (o) return {o->plane, o->pitch, o->width, o->height};
    return ol->images[i];
}
// The format of frames in either form, and how many descriptions they hold
template <class Batch, class List>
static int frameFormat(const Batch* b, const List* l) {
    return b ? b->format : l->format;
}
template <class List>
static int frameCount(const void* b, const List* l) {
    return b ? 1 : l->count;
}

// The planes of frame image m: each pitch at least its row's bytes, each plane device or managed memory of `device`; P010's 16-bit
// samples also need even pitches and image strides and 2-byte-aligned planes.
static int checkFramePlanes(const char* api, const char* what, const snnb_frames& m, int device) {
    const bool p010 = m.format == SNNB_FRAME_P010;
    for (int p = 0; p < 3; ++p) {
        const long long row = frameRowBytes(m.format, m.width, p);
        if (!row) continue;
        SNNB_REQUIRE(m.pitch[p] >= row, "%s: %s %d: pitch %d is less than its row's %lld bytes", api, what, p, m.pitch[p], row);
        SNNB_REQUIRE(!p010 || (m.pitch[p] % 2 == 0 && m.image_stride[p] % 2 == 0), "%s: %s %d: P010 pitch %d and image stride %lld must be even", api, what, p,
                     m.pitch[p], m.image_stride[p]);
        if (int rc = checkDevicePointer(api, m.plane[p], p010 ? 2 : 1, device, what, p)) return rc;
    }
    return 0;
}

// A caller's stream that work may be ordered on: NULL (the context's), or a stream that is not being captured.
static int checkCallerStream(const char* api, cudaStream_t stream) {
    if (stream) {
        cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
        const cudaError_t e = cudaStreamIsCapturing(stream, &cap);
        if (e != cudaSuccess) cudaGetLastError();
        SNNB_REQUIRE(e == cudaSuccess, "%s: stream %p: %s", api, (void*) stream, cudaGetErrorString(e));
        SNNB_REQUIRE(cap == cudaStreamCaptureStatusNone, "%s: stream %p is being captured; capture into the caller's CUDA graph is not supported", api, (void*) stream);
    }
    return 0;
}

// The matrix (YUV formats) and size of one frame description. `image` prefixes each message: "" for an snnb_frames batch, "image 3: "
// for entry 3 of a frame list.
static int checkFrameImage(const char* api, const char* image, const snnb_frames& m) {
    if (m.format != SNNB_FRAME_RGBA8) {
        const int base = m.matrix & ~SNNB_YUV_FULL_RANGE;
        SNNB_REQUIRE(base == SNNB_YUV_BT601 || base == SNNB_YUV_BT709 || base == SNNB_YUV_BT2020, "%s: %sunknown YUV matrix %d", api, image, m.matrix);
        SNNB_REQUIRE(base == SNNB_YUV_BT601 || !(m.matrix & SNNB_YUV_FULL_RANGE), "%s: %sYUV matrix %d: full range is defined for BT.601 only", api, image,
                     m.matrix);
    }
    SNNB_REQUIRE(m.width >= 1 && m.height >= 1, "%s: %sframe size %d x %d; width and height must be >= 1", api, image, m.width, m.height);
    return 0;
}

int MixedInferenceCore::checkDeviceFeed(const char* api, const DeviceFeed& in, cudaStream_t stream) {
    if (in.frames || in.list) {
        // one snnb_frames (its batch shares one description) or each image of a list, in run_frames' order of checks: the format,
        // each image's matrix and size, the model's input, then each image's planes
        const int format = frameFormat(in.frames, in.list);
        SNNB_REQUIRE(knownFrameFormat(format), "%s: unknown frame format %d", api, format);
        if (in.list) {
            SNNB_REQUIRE(in.list->images, "%s: null images", api);
            const int n = in.list->count;
            if (in.rois)
                SNNB_REQUIRE(n >= 1 && n <= SNNB_FRAME_LIST_MAX, "%s: count %d; a list holds 1 to %d frames", api, n, (int) SNNB_FRAME_LIST_MAX);
            else
                SNNB_REQUIRE(n == curBatch && n <= SNNB_FRAME_LIST_MAX, "%s: count %d; the list must hold the model's batch of %d images (at most %d)", api, n,
                             curBatch, (int) SNNB_FRAME_LIST_MAX);
        }
        const int images = frameCount(in.frames, in.list);
        char image[32] = "", planes[32] = "plane";
        for (int i = 0; i < images; ++i) {
            if (in.list) std::snprintf(image, sizeof(image), "image %d: ", i);
            if (int rc = checkFrameImage(api, image, frameImage(in.frames, in.list, i))) return rc;
        }
        SNNB_REQUIRE(inputLayers.size() == 1, "%s: the model has %d inputs; frames feed a model with exactly one", api, (int) inputLayers.size());
        const snnb_tensor* t = inputLayers[0]->output;
        SNNB_REQUIRE(t->c >= 1 && t->c <= 4, "%s: the model input has %d channels; frames feed 1 to 4 (RGBA components)", api, t->c);
        if (in.luma) {
            SNNB_REQUIRE(format != SNNB_FRAME_RGBA8, "%s: RGBA8 frames have no Y plane; luma input takes NV12, NV21, I420 or P010 frames", api);
            SNNB_REQUIRE(t->c == 1, "%s: the model input has %d channels; the Y plane feeds exactly 1", api, t->c);
        }
        for (int i = 0; i < images; ++i) {
            if (in.list) std::snprintf(planes, sizeof(planes), "image %d plane", i);
            if (int rc = checkFramePlanes(api, planes, frameImage(in.frames, in.list, i), ctx->device)) return rc;
        }
        if (in.rois) {
            SNNB_REQUIRE(in.numFrames >= 1, "%s: num_frames %d; at least one frame is required", api, in.numFrames);
            SNNB_REQUIRE(options.batch <= 65535, "%s: batch %u; regions fill at most 65535 slots", api, options.batch);
            if (int rc = checkDevicePointer(api, in.rois, sizeof(int), ctx->device, "rois", 0)) return rc;
            if (in.roiCount)
                if (int rc = checkDevicePointer(api, in.roiCount, sizeof(int), ctx->device, "count", 0)) return rc;
        }
    } else {
        SNNB_REQUIRE(in.inputs, "%s: null inputs", api);
        SNNB_REQUIRE(in.numInputs == (int) inputLayers.size(), "%s: %d inputs given, the model has %d", api, in.numInputs, (int) inputLayers.size());
        for (int i = 0; i < in.numInputs; ++i)
            if (int rc = checkDeviceBuffer(api, in.inputs[i], ctx->device, "input", i)) return rc;
    }
    return checkCallerStream(api, stream);
}

// f(*in.frames) or f(*in.list): each frame launcher has an overload for either form
template <class Feed, class F>
static int withFrames(const Feed& in, F&& f) {
    if (in.list) return f(*in.list);
    return f(*in.frames);
}

// The caller's stream -> the context's stream, the input staging and the forward pass. Called after every check has passed.
int MixedInferenceCore::enqueueDeviceForward(const DeviceFeed& in, cudaStream_t stream) {
    if (!callerReady) SNNB_CUDA_OK(cudaEventCreateWithFlags(&callerReady, cudaEventDisableTiming));
    if (!deviceDone) SNNB_CUDA_OK(cudaEventCreateWithFlags(&deviceDone, cudaEventDisableTiming));
    if (stream && stream != ctx->stream) { // a stream of another device fails here, before anything is launched
        SNNB_CUDA_OK(cudaEventRecord(callerReady, stream));
        SNNB_CUDA_OK(cudaStreamWaitEvent(ctx->stream, callerReady, 0));
    }
    snnb_tensor* t = inputLayers[0]->output;
    if (in.frames || in.list) {
        const int rc = withFrames(in, [&](const auto& fr) {
            return in.rois ? launch_frame_roi_input(ctx, fr, in.numFrames, in.rois, in.roiCount, t) : launch_frame_input(ctx, fr, t, in.luma);
        });
        if (rc) return 1;
    } else {
        for (int i = 0; i < in.numInputs; ++i)
            if (launch_device_input(ctx, in.inputs[i], inputLayers[i]->output)) return 1;
    }
    return counted(in) ? forwardCounted(in.roiCount) : forward();
}

// The context's stream -> the caller's: work enqueued on `stream` from now on sees everything enqueued above.
int MixedInferenceCore::fenceToCaller(cudaStream_t stream) {
    if (stream && stream != ctx->stream) {
        SNNB_CUDA_OK(cudaEventRecord(deviceDone, ctx->stream));
        SNNB_CUDA_OK(cudaStreamWaitEvent(stream, deviceDone, 0));
    }
    return 0;
}

int MixedInferenceCore::runDevice(const snnb_device_buffer* inputs, int numInputs, const snnb_device_buffer* outputs, int numOutputs, int* classes1Dev,
                                  cudaStream_t stream) {
    DeviceFeed in;
    in.inputs = inputs, in.numInputs = numInputs;
    return runDeviceFeed("snnb_model_run_device", in, outputs, numOutputs, classes1Dev, stream);
}
int MixedInferenceCore::runFrames(const snnb_frames* frames, const snnb_device_buffer* outputs, int numOutputs, int* classes1Dev, cudaStream_t stream) {
    SNNB_REQUIRE(frames, "snnb_model_run_frames: null frames");
    DeviceFeed in;
    in.frames = frames;
    return runDeviceFeed("snnb_model_run_frames", in, outputs, numOutputs, classes1Dev, stream);
}
int MixedInferenceCore::runRois(const snnb_frames* frames, int numFrames, const snnb_roi* roisDev, const int* countDev, const snnb_device_buffer* outputs,
                                int numOutputs, int* classes1Dev, cudaStream_t stream) {
    SNNB_REQUIRE(frames, "snnb_model_run_rois: null frames");
    SNNB_REQUIRE(roisDev, "snnb_model_run_rois: null rois");
    DeviceFeed in;
    in.frames = frames, in.rois = roisDev, in.roiCount = countDev, in.numFrames = numFrames;
    return runDeviceFeed("snnb_model_run_rois", in, outputs, numOutputs, classes1Dev, stream);
}
int MixedInferenceCore::runFrameList(const snnb_frame_list* frames, const snnb_device_buffer* outputs, int numOutputs, int* classes1Dev, cudaStream_t stream) {
    SNNB_REQUIRE(frames, "snnb_model_run_frame_list: null frames");
    DeviceFeed in;
    in.list = frames;
    return runDeviceFeed("snnb_model_run_frame_list", in, outputs, numOutputs, classes1Dev, stream);
}
int MixedInferenceCore::runRoisList(const snnb_frame_list* frames, const snnb_roi* roisDev, const int* countDev, const snnb_device_buffer* outputs,
                                    int numOutputs, int* classes1Dev, cudaStream_t stream) {
    SNNB_REQUIRE(frames, "snnb_model_run_rois_list: null frames");
    SNNB_REQUIRE(roisDev, "snnb_model_run_rois_list: null rois");
    DeviceFeed in;
    in.list = frames, in.rois = roisDev, in.roiCount = countDev, in.numFrames = frames->count;
    return runDeviceFeed("snnb_model_run_rois_list", in, outputs, numOutputs, classes1Dev, stream);
}

// A counted region call (counted(in)): refused while the context's stream is being captured; otherwise the current batch's dispatch graph,
// built on the first such call. Nothing to do for any other call.
int MixedInferenceCore::prepareCounted(const char* api, const DeviceFeed& in) {
    if (!counted(in)) return 0;
    cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
    SNNB_CUDA_OK(cudaStreamIsCapturing(ctx->stream, &cap));
    SNNB_REQUIRE(cap == cudaStreamCaptureStatusNone,
                 "%s: the context's stream is being captured (snnb_graph_capture_begin); a call with a device-side count and declared sizes runs "
                 "a graph with conditional nodes, which cannot become part of another graph",
                 api);
    return !cur->dispatchExec && buildDispatch(api, in.roiCount) ? 1 : 0;
}

int MixedInferenceCore::runDeviceFeed(const char* api, const DeviceFeed& in, const snnb_device_buffer* outputs, int numOutputs, int* classes1Dev,
                                      cudaStream_t stream) {
    // everything is validated before the first enqueue: a refused call leaves no work behind
    SNNB_REQUIRE(numOutputs >= 0 && numOutputs <= (int) outputLayers.size(), "%s: %d outputs requested, the model has %d", api, numOutputs,
                 (int) outputLayers.size());
    SNNB_REQUIRE(outputs || numOutputs == 0, "%s: null outputs", api);
    SNNB_REQUIRE(!(in.rois && outputLayers[0]->typeName == "YOLO"),
                 "%s: output 0 is a YOLO detection list; detection on regions is not supported by this call: use %s", api,
                 in.list ? "snnb_model_detect_rois_list" : "snnb_model_detect_rois");
    SNNB_REQUIRE(outputLayers[0]->typeName != "YOLO",
                 "%s: output 0 is a YOLO detection list; use %s for device detections, or snnb_model_run or "
                 "snnb_model_submit / snnb_model_wait and read the boxes with snnb_model_get_boxes",
                 api, in.list ? "snnb_model_detect_frame_list" : (in.frames ? "snnb_model_detect_frames" : "snnb_model_detect_device"));
    if (int rc = checkDeviceFeed(api, in, stream)) return rc;
    const int device = ctx->device;
    for (int j = 0; j < numOutputs; ++j) {
        if (!outputs[j].data) continue;
        SNNB_REQUIRE(outputLayers[j]->output, "%s: output %d (%s) has no device tensor", api, j, outputLayers[j]->name.c_str());
        if (int rc = checkDeviceBuffer(api, outputs[j], device, "output", j)) return rc;
    }
    if (classes1Dev) {
        SNNB_REQUIRE(isClassifier, "%s: classes requested, but the model is not a classifier (output 0 is not 1 x 1 x C with C > 1)", api);
        if (int rc = checkDevicePointer(api, classes1Dev, sizeof(int), device, "classes", 0)) return rc;
    }
    if (int rc = prepareCounted(api, in)) return rc;

    if (enqueueDeviceForward(in, stream)) return 1;
    for (int j = 0; j < numOutputs; ++j)
        if (outputs[j].data && launch_device_output(ctx, outputLayers[j]->output, outputs[j])) return 1;
    if (classes1Dev && launch_argmax(ctx, outputLayers[0]->output, classes1Dev, 1)) return 1; // core.cpp:228-233: argmax + 1
    if (in.rois) { // the slots without a valid region: every output byte and the class zero
        const int B = curBatch;
        auto clear = [&](void* dst, long long slotBytes) {
            return withFrames(in, [&](const auto& fr) { return launch_roi_clear(ctx, fr, in.numFrames, in.rois, in.roiCount, B, dst, slotBytes); });
        };
        for (int j = 0; j < numOutputs; ++j) {
            if (!outputs[j].data) continue;
            const snnb_tensor* t = outputLayers[j]->output;
            const long long elem = outputs[j].dtype == SNNB_DTYPE_F32 ? 4 : (outputs[j].dtype == SNNB_DTYPE_F16 ? 2 : 1);
            if (clear(outputs[j].data, (long long) t->h * t->w * t->c * elem)) return 1;
        }
        if (classes1Dev && clear(classes1Dev, (long long) sizeof(int))) return 1;
    }
    return fenceToCaller(stream);
}

// Detections in device memory: the forward pass, then the whole YOLO decode (threshold, stable score sort, NMS) in three kernels.
// Reads the heads only: the host detection lists (`boxes`) and the candidate buffers of run() / submit() are not touched.
int MixedInferenceCore::detectDevice(const snnb_device_buffer* inputs, int numInputs, float* rowsDev, int maxRows, int* countsDev, cudaStream_t stream) {
    DeviceFeed in;
    in.inputs = inputs, in.numInputs = numInputs;
    return detectDeviceFeed("snnb_model_detect_device", in, rowsDev, maxRows, countsDev, stream);
}
int MixedInferenceCore::detectFrames(const snnb_frames* frames, float* rowsDev, int maxRows, int* countsDev, cudaStream_t stream) {
    SNNB_REQUIRE(frames, "snnb_model_detect_frames: null frames");
    DeviceFeed in;
    in.frames = frames;
    return detectDeviceFeed("snnb_model_detect_frames", in, rowsDev, maxRows, countsDev, stream);
}
int MixedInferenceCore::detectFrameList(const snnb_frame_list* frames, float* rowsDev, int maxRows, int* countsDev, cudaStream_t stream) {
    SNNB_REQUIRE(frames, "snnb_model_detect_frame_list: null frames");
    DeviceFeed in;
    in.list = frames;
    return detectDeviceFeed("snnb_model_detect_frame_list", in, rowsDev, maxRows, countsDev, stream);
}

int MixedInferenceCore::detectDeviceFeed(const char* api, const DeviceFeed& in, float* rowsDev, int maxRows, int* countsDev, cudaStream_t stream) {
    SNNB_REQUIRE(yolo, "%s: the model has no YOLO output; use %s", api,
                 in.list ? "snnb_model_run_frame_list" : (in.frames ? "snnb_model_run_frames" : "snnb_model_run_device"));
    if (int rc = checkDetectOutputs(api, in, rowsDev, maxRows, countsDev, stream)) return rc;

    if (enqueueDeviceForward(in, stream)) return 1;
    if (launch_yolo_detect(ctx, yolo->inputs[0], yolo->inputs[1], detectScratch, maxRows, rowsDev, countsDev)) return 1;
    return fenceToCaller(stream);
}

// The checks the detecting calls share once the model is known to have a YOLO output: max_rows, the feed, rows and counts, the heads;
// then the decode's scratch (sized for the loaded batch, whatever the model's batch is now), allocated on first use.
int MixedInferenceCore::checkDetectOutputs(const char* api, const DeviceFeed& in, float* rowsDev, int maxRows, int* countsDev, cudaStream_t stream) {
    SNNB_REQUIRE(maxRows >= 1 && maxRows <= 100, "%s: max_rows %d is outside 1..100", api, maxRows);
    if (int rc = checkDeviceFeed(api, in, stream)) return rc;
    if (int rc = checkDevicePointer(api, rowsDev, sizeof(float), ctx->device, "rows", 0)) return rc;
    if (int rc = checkDevicePointer(api, countsDev, sizeof(int), ctx->device, "counts", 0)) return rc;
    SNNB_REQUIRE(yolo->inputs.size() == 2 && yolo->inputs[0]->c >= 18 && yolo->inputs[1]->c >= 18, "%s: %s: YOLO expects two heads of >= 18 channels", api,
                 yolo->name.c_str());
    if (!detectScratch) {
        snnb_tensor h0 = *yolo->inputs[0], h1 = *yolo->inputs[1];
        h0.n = h1.n = (int) options.batch;
        SNNB_CUDA_OK(cudaMalloc(&detectScratch, yolo_detect_scratch_bytes(&h0, &h1)));
    }
    return 0;
}

// Detection on regions: runRois' input staging and forward pass (the dispatch graph for a counted call), the device decode of every slot
// into roiScratch (100 rows per slot, as detectFrames with max_rows 100), then the merge: each valid slot's rows mapped to its frame,
// one stable score sort and one greedy NMS per frame, into the caller's rows and counts.
int MixedInferenceCore::detectRois(const snnb_frames* frames, int numFrames, const snnb_roi* roisDev, const int* countDev, float* rowsDev, int maxRows,
                                   int* countsDev, cudaStream_t stream) {
    SNNB_REQUIRE(frames, "snnb_model_detect_rois: null frames");
    SNNB_REQUIRE(roisDev, "snnb_model_detect_rois: null rois");
    DeviceFeed in;
    in.frames = frames, in.rois = roisDev, in.roiCount = countDev, in.numFrames = numFrames;
    return detectRoisFeed("snnb_model_detect_rois", in, rowsDev, maxRows, countsDev, stream);
}
int MixedInferenceCore::detectRoisList(const snnb_frame_list* frames, const snnb_roi* roisDev, const int* countDev, float* rowsDev, int maxRows, int* countsDev,
                                       cudaStream_t stream) {
    SNNB_REQUIRE(frames, "snnb_model_detect_rois_list: null frames");
    SNNB_REQUIRE(roisDev, "snnb_model_detect_rois_list: null rois");
    DeviceFeed in;
    in.list = frames, in.rois = roisDev, in.roiCount = countDev, in.numFrames = frames->count;
    return detectRoisFeed("snnb_model_detect_rois_list", in, rowsDev, maxRows, countsDev, stream);
}
int MixedInferenceCore::detectRoisFeed(const char* api, const DeviceFeed& in, float* rowsDev, int maxRows, int* countsDev, cudaStream_t stream) {
    SNNB_REQUIRE(yolo, "%s: the model has no YOLO output; use %s", api, in.list ? "snnb_model_run_rois_list" : "snnb_model_run_rois");
    if (int rc = checkDetectOutputs(api, in, rowsDev, maxRows, countsDev, stream)) return rc;
    if (int rc = prepareCounted(api, in)) return rc;
    const int B             = (int) options.batch;
    const size_t rowsBytes  = (size_t) B * 100 * 6 * sizeof(float);
    const size_t countBytes = ((size_t) B * sizeof(int) + 255) & ~(size_t) 255;
    const size_t mergeBytes = roi_merge_scratch_bytes(B);
    if (in.numFrames > roiSegsCap) { // at least 256 frames; a larger call replaces the scratch once the work that reads it is done
        if (roiScratch) {
            SNNB_CUDA_OK(cudaStreamSynchronize(ctx->stream));
            cudaFree(roiScratch);
            roiScratch = nullptr, roiSegsCap = 0;
        }
        const int cap = std::max(in.numFrames, (int) SNNB_FRAME_LIST_MAX);
        SNNB_CUDA_OK(cudaMalloc(&roiScratch, rowsBytes + countBytes + mergeBytes + (size_t) cap * 2 * sizeof(int)));
        roiSegsCap = cap;
    }
    char* base      = static_cast<char*>(roiScratch);
    float* slotRows = reinterpret_cast<float*>(base);
    int* slotCounts = reinterpret_cast<int*>(base + rowsBytes);
    void* merge     = base + rowsBytes + countBytes;
    void* segs      = base + rowsBytes + countBytes + mergeBytes;

    if (enqueueDeviceForward(in, stream)) return 1;
    if (launch_yolo_detect(ctx, yolo->inputs[0], yolo->inputs[1], detectScratch, 100, slotRows, slotCounts)) return 1;
    const int rc = withFrames(in, [&](const auto& fr) {
        return launch_roi_merge(ctx, fr, in.numFrames, in.rois, in.roiCount, curBatch, slotRows, slotCounts, merge, segs, maxRows, rowsDev, countsDev);
    });
    if (rc) return 1;
    return fenceToCaller(stream);
}

// The out frames of transform / transform_luma: one snnb_frames_out, or (ol) each image of an output list, which must hold one image per
// frame of the input list. Each size, then each image's planes, in transform_frames' order of checks; list errors name the image.
static int checkFramesOut(const char* api, const snnb_frames_out* o, const snnb_frame_out_list* ol, int frames, int device) {
    if (ol) {
        SNNB_REQUIRE(ol->images, "%s: null out images", api);
        SNNB_REQUIRE(ol->count == frames, "%s: out count %d; the out list must hold one image per frame (%d)", api, ol->count, frames);
    }
    char image[32] = "", planes[40] = "out plane";
    for (int i = 0; i < frameCount(o, ol); ++i) {
        if (ol) std::snprintf(image, sizeof(image), "image %d: ", i), std::snprintf(planes, sizeof(planes), "image %d out plane", i);
        const snnb_frames m = frameImage(o, ol, i);
        SNNB_REQUIRE(m.width >= 1 && m.height >= 1, "%s: %sout frame size %d x %d; width and height must be >= 1", api, image, m.width, m.height);
        if (int rc = checkFramePlanes(api, planes, m, device)) return rc;
    }
    return 0;
}

// Frames in, frames out: runFrames' input staging and forward pass, then output 0 quantised, resized and colour-converted into `out` in
// one kernel. The output kernel runs after the forward pass on the context's stream, so `out` may alias the input frames.
int MixedInferenceCore::transformFrames(const snnb_frames* frames, const snnb_frames_out* out, cudaStream_t stream) {
    SNNB_REQUIRE(frames, "snnb_model_transform_frames: null frames");
    SNNB_REQUIRE(out, "snnb_model_transform_frames: null out");
    DeviceFeed in;
    in.frames = frames;
    return transformDeviceFeed("snnb_model_transform_frames", in, out, nullptr, stream);
}
int MixedInferenceCore::transformFrameList(const snnb_frame_list* frames, const snnb_frame_out_list* out, cudaStream_t stream) {
    SNNB_REQUIRE(frames, "snnb_model_transform_frame_list: null frames");
    SNNB_REQUIRE(out, "snnb_model_transform_frame_list: null out");
    DeviceFeed in;
    in.list = frames;
    return transformDeviceFeed("snnb_model_transform_frame_list", in, nullptr, out, stream);
}
int MixedInferenceCore::transformDeviceFeed(const char* api, const DeviceFeed& in, const snnb_frames_out* o, const snnb_frame_out_list* ol, cudaStream_t stream) {
    if (int rc = checkDeviceFeed(api, in, stream)) return rc;
    const int format = frameFormat(o, ol);
    SNNB_REQUIRE(knownFrameFormat(format), "%s: unknown out frame format %d", api, format);
    if (int rc = checkFramesOut(api, o, ol, frameCount(in.frames, in.list), ctx->device)) return rc;
    SNNB_REQUIRE(outputLayers[0]->typeName != "YOLO", "%s: output 0 is a YOLO detection list; frames are written from an image output", api);
    const snnb_tensor* t = outputLayers[0]->output;
    SNNB_REQUIRE(t, "%s: output 0 (%s) has no device tensor", api, outputLayers[0]->name.c_str());
    SNNB_REQUIRE(t->c == 1 || t->c == 3 || t->c == 4, "%s: output 0 has %d channels; frames are written from 1 (grey), 3 (RGB) or 4 (RGBA)", api, t->c);

    if (enqueueDeviceForward(in, stream)) return 1;
    if (o ? launch_frame_output(ctx, t, *o) : launch_frame_output(ctx, t, *ol)) return 1;
    return fenceToCaller(stream);
}

// The bytes plane p of `n` images of m spans, from its first image's first byte to its last image's last row byte; false for an unused plane
static bool planeExtent(const snnb_frames& m, int n, int p, uintptr_t& begin, uintptr_t& end) {
    const long long row = frameRowBytes(m.format, m.width, p);
    if (!row) return false;
    const long long rows = p == 0 ? m.height : (m.height + 1) / 2, span = (long long) (n - 1) * m.image_stride[p];
    begin = reinterpret_cast<uintptr_t>(m.plane[p]) + (span < 0 ? span : 0);
    end   = reinterpret_cast<uintptr_t>(m.plane[p]) + (span > 0 ? span : 0) + (rows - 1) * m.pitch[p] + row;
    return true;
}

// Luma frames in, luma frames out: the Y plane feeds a 1-channel model, output 0 (1 channel) becomes the Y plane of `out`, and the same
// output kernel resamples the source frames' chroma into out's chroma. The kernel reads the source chroma while it writes, so out must
// keep clear of it unless out is the source frames themselves (each chroma sample is then read and written by one thread). A list runs
// every image in one kernel: out image i may be source image i itself, and must keep clear of every other image's source chroma.
int MixedInferenceCore::transformLuma(const snnb_frames* frames, const snnb_frames_out* out, cudaStream_t stream) {
    SNNB_REQUIRE(frames, "snnb_model_transform_luma: null frames");
    SNNB_REQUIRE(out, "snnb_model_transform_luma: null out");
    DeviceFeed in;
    in.frames = frames, in.luma = true;
    return transformLumaDeviceFeed("snnb_model_transform_luma", in, out, nullptr, stream);
}
int MixedInferenceCore::transformLumaList(const snnb_frame_list* frames, const snnb_frame_out_list* out, cudaStream_t stream) {
    SNNB_REQUIRE(frames, "snnb_model_transform_luma_list: null frames");
    SNNB_REQUIRE(out, "snnb_model_transform_luma_list: null out");
    DeviceFeed in;
    in.list = frames, in.luma = true;
    return transformLumaDeviceFeed("snnb_model_transform_luma_list", in, nullptr, out, stream);
}
int MixedInferenceCore::transformLumaDeviceFeed(const char* api, const DeviceFeed& in, const snnb_frames_out* o, const snnb_frame_out_list* ol,
                                                cudaStream_t stream) {
    if (int rc = checkDeviceFeed(api, in, stream)) return rc;
    const int format = frameFormat(in.frames, in.list), oformat = frameFormat(o, ol);
    SNNB_REQUIRE(knownFrameFormat(oformat), "%s: unknown out frame format %d", api, oformat);
    SNNB_REQUIRE(oformat != SNNB_FRAME_RGBA8, "%s: out format RGBA8 has no Y plane; luma frames are written as NV12, NV21, I420 or P010", api);
    SNNB_REQUIRE((oformat == SNNB_FRAME_P010) == (format == SNNB_FRAME_P010),
                 "%s: frames format %d, out format %d: the bit depths differ; P010 frames are written from P010 frames only", api, format, oformat);
    const int images = frameCount(in.frames, in.list);
    if (int rc = checkFramesOut(api, o, ol, images, ctx->device)) return rc;
    SNNB_REQUIRE(outputLayers[0]->typeName != "YOLO", "%s: output 0 is a YOLO detection list; frames are written from an image output", api);
    const snnb_tensor* t = outputLayers[0]->output;
    SNNB_REQUIRE(t, "%s: output 0 (%s) has no device tensor", api, outputLayers[0]->name.c_str());
    SNNB_REQUIRE(t->c == 1, "%s: output 0 has %d channels; the Y plane is written from exactly 1", api, t->c);
    // out image i against source image j: a batch spans the model's batch at its image strides, a list image itself
    char oname[24] = "", sname[24] = "";
    for (int i = 0; i < images; ++i) {
        const snnb_frames out = frameImage(o, ol, i), own = frameImage(in.frames, in.list, i);
        bool same = out.format == own.format && out.width == own.width && out.height == own.height;
        for (int p = 0; p < 3 && same; ++p)
            if (frameRowBytes(format, own.width, p))
                same = out.plane[p] == own.plane[p] && out.pitch[p] == own.pitch[p] && out.image_stride[p] == own.image_stride[p];
        for (int j = 0; j < images; ++j) {
            if (j == i && same) continue;
            if (in.list) std::snprintf(oname, sizeof(oname), "image %d ", i), std::snprintf(sname, sizeof(sname), "image %d ", j);
            const snnb_frames src = frameImage(in.frames, in.list, j);
            for (int p = 0; p < 3; ++p) {
                uintptr_t ob, oe;
                if (!planeExtent(out, curBatch, p, ob, oe)) continue;
                for (int q = 1; q < 3; ++q) {
                    uintptr_t sb, se;
                    if (!planeExtent(src, curBatch, q, sb, se)) continue;
                    SNNB_REQUIRE(oe <= sb || se <= ob,
                                 "%s: %sout plane %d overlaps %ssource chroma plane %d; out may alias the source chroma only as the source frames themselves", api,
                                 oname, p, sname, q);
                }
            }
        }
    }

    if (enqueueDeviceForward(in, stream)) return 1;
    if (o ? launch_luma_output(ctx, t, *in.frames, *o) : launch_luma_output(ctx, t, *in.list, *ol)) return 1;
    return fenceToCaller(stream);
}

// Frames in, labels out: runFrames' (or, with luma, transformLuma's) input staging and forward pass, then output 0's scores resampled
// to the label plane and reduced to one byte per pixel in one kernel. The kernel reads only the model's tensor, so the plane may alias
// the input frames.
int MixedInferenceCore::segmentFrames(const snnb_frames* frames, bool luma, const snnb_labels_out* out, cudaStream_t stream) {
    SNNB_REQUIRE(frames, "snnb_model_segment_frames: null frames");
    SNNB_REQUIRE(out, "snnb_model_segment_frames: null out");
    DeviceFeed in;
    in.frames = frames, in.luma = luma;
    return segmentDeviceFeed("snnb_model_segment_frames", in, out, nullptr, stream);
}
int MixedInferenceCore::segmentFrameList(const snnb_frame_list* frames, bool luma, const snnb_labels_list* out, cudaStream_t stream) {
    SNNB_REQUIRE(frames, "snnb_model_segment_frame_list: null frames");
    SNNB_REQUIRE(out, "snnb_model_segment_frame_list: null out");
    DeviceFeed in;
    in.list = frames, in.luma = luma;
    return segmentDeviceFeed("snnb_model_segment_frame_list", in, nullptr, out, stream);
}
int MixedInferenceCore::segmentDeviceFeed(const char* api, const DeviceFeed& in, const snnb_labels_out* o, const snnb_labels_list* ol, cudaStream_t stream) {
    if (int rc = checkDeviceFeed(api, in, stream)) return rc;
    if (ol) {
        SNNB_REQUIRE(ol->images, "%s: null out images", api);
        SNNB_REQUIRE(ol->count == in.list->count, "%s: out count %d; the out list must hold one image per frame (%d)", api, ol->count, in.list->count);
    }
    char image[32] = "", plane[40] = "label plane";
    for (int i = 0; i < frameCount(o, ol); ++i) {
        if (ol) std::snprintf(image, sizeof(image), "image %d: ", i), std::snprintf(plane, sizeof(plane), "image %d label plane", i);
        const snnb_labels_image m = labelsImage(o, ol, i);
        SNNB_REQUIRE(m.width >= 1 && m.height >= 1, "%s: %slabel plane size %d x %d; width and height must be >= 1", api, image, m.width, m.height);
        SNNB_REQUIRE(m.pitch >= m.width, "%s: %slabel plane pitch %d is less than its width %d", api, image, m.pitch, m.width);
        if (int rc = checkDevicePointer(api, m.plane, 1, ctx->device, plane, 0)) return rc;
    }
    SNNB_REQUIRE(outputLayers[0]->typeName != "YOLO", "%s: output 0 is a YOLO detection list; labels are written from per-pixel class scores", api);
    const snnb_tensor* t = outputLayers[0]->output;
    SNNB_REQUIRE(t, "%s: output 0 (%s) has no device tensor", api, outputLayers[0]->name.c_str());
    SNNB_REQUIRE(t->c >= 1 && t->c <= 256, "%s: output 0 has %d channels; an 8-bit label plane is written from 1 to 256", api, t->c);

    if (enqueueDeviceForward(in, stream)) return 1;
    if (o ? launch_segment_output(ctx, t, *o) : launch_segment_output(ctx, t, *ol)) return 1;
    return fenceToCaller(stream);
}

int MixedInferenceCore::layerOutput(int layerId, float* host, size_t capacityFloats) {
    SNNB_REQUIRE(layerId >= 0 && layerId < (int) layers.size() && host, "layerOutput: bad argument");
    GenericModelLayer* L = layers[layerId].get();
    SNNB_REQUIRE(L->output, "layerOutput: layer %d (%s) has no device tensor", layerId, L->name.c_str());
    SNNB_REQUIRE(!(L->typeName == "Conv2D" && static_cast<Conv2DLayer*>(L)->fusedAct >= 0),
                 "layerOutput: layer %d (%s) was fused into its Add; load the model with fuse=0 to observe it", layerId, L->name.c_str());
    SNNB_REQUIRE(!(L->fusedAway && L->typeName == "AveragePooling2D"),
                 "layerOutput: layer %d (%s) was fused into the classifier head (pool + Dense in one launch); load the model with fuse=0 to observe it", layerId,
                 L->name.c_str());
    const size_t floats = L->output->pixels() * L->output->c;
    SNNB_REQUIRE(capacityFloats >= floats, "layerOutput: buffer too small (%zu < %zu floats)", capacityFloats, floats);
    return snnb_tensor_download_nhwc(ctx, L->output, host);
}

int MixedInferenceCore::timeLayers(std::vector<float>& ms) {
    ms.assign(layers.size(), 0.0f);
    std::vector<cudaEvent_t> ev(graph.sorted.size() + 1);
    for (auto& e : ev) SNNB_CUDA_OK(cudaEventCreate(&e));
    SNNB_CUDA_OK(cudaEventRecord(ev[0], ctx->stream));
    layerKernels.assign(layers.size(), std::string());
    for (size_t i = 0; i < graph.sorted.size(); ++i) {
        GenericModelLayer* L = graph.sorted[i];
        if (!(L->fusedAway || L->isInputLayer || L->typeName == "YOLO")) {
            ctx->last_kernel = nullptr;
            if (int rc = L->run(ctx)) return rc;
            layerKernels[L->layerId] = ctx->last_kernel ? ctx->last_kernel : (L->typeName + " kernels");
        }
        SNNB_CUDA_OK(cudaEventRecord(ev[i + 1], ctx->stream));
    }
    SNNB_CUDA_OK(cudaStreamSynchronize(ctx->stream));
    for (size_t i = 0; i < graph.sorted.size(); ++i) {
        float t = 0;
        SNNB_CUDA_OK(cudaEventElapsedTime(&t, ev[i], ev[i + 1]));
        ms[graph.sorted[i]->layerId] = t;
    }
    for (auto& e : ev) cudaEventDestroy(e);
    return 0;
}

int MixedInferenceCore::dumpOutputs(const std::string& dir) {
    for (auto& l : layers) {
        if (!l->output || l->fusedAway) continue;
        // a Conv2D fused into its Add writes the ADD's tensor (post-add, post-activation): under the conv's name the file would
        // not be what a reference run dumps for that layer (layerOutput() refuses the same case)
        SNNB_REQUIRE(!(l->typeName == "Conv2D" && l->fusedAct >= 0), "dumpOutputs: %s was fused into its Add; load the model with fuse=0 to dump every layer", l->name.c_str());
        std::string path = dir + "/" + l->name + " pass[0].dump"; // vulkanBackend.cpp:108-143 naming
        if (snnb_tensor_dump(ctx, l->output, path.c_str())) return 1;
    }
    return 0;
}

} // namespace snn

// snnb_rois_from_detections and its per-frame-size form: context-level calls with no model state, so their one kernel runs on the
// caller's stream itself. frameWh == nullptr: every frame is fw x fh; else frame n is frameWh[2n] x frameWh[2n + 1].
static int roisFromDetections(const char* api, snnb_context* ctx, const float* rows, const int* counts, int numFrames, int maxRows, int fw, int fh,
                              const int* frameWh, const snnb_roi_select* sel, snnb_roi* rois, int capacity, int* count, cudaStream_t stream) {
    SNNB_REQUIRE(sel, "%s: null sel", api);
    SNNB_REQUIRE(numFrames >= 1, "%s: num_frames %d; at least one frame is required", api, numFrames);
    SNNB_REQUIRE(maxRows >= 1 && maxRows <= 100, "%s: max_rows %d is outside 1..100", api, maxRows);
    SNNB_REQUIRE((long long) numFrames * maxRows <= 0x7fffffffLL, "%s: %d frames of %d rows", api, numFrames, maxRows);
    if (frameWh) {
        SNNB_REQUIRE(numFrames <= SNNB_FRAME_LIST_MAX, "%s: num_frames %d is more than %d", api, numFrames, (int) SNNB_FRAME_LIST_MAX);
        for (int n = 0; n < numFrames; ++n)
            SNNB_REQUIRE(frameWh[2 * n] >= 1 && frameWh[2 * n + 1] >= 1, "%s: frame %d: size %d x %d; width and height must be >= 1", api, n, frameWh[2 * n],
                         frameWh[2 * n + 1]);
    } else {
        SNNB_REQUIRE(fw >= 1 && fh >= 1, "%s: frame size %d x %d; width and height must be >= 1", api, fw, fh);
    }
    SNNB_REQUIRE(capacity >= 1, "%s: capacity %d; at least one region is required", api, capacity);
    SNNB_REQUIRE(std::isfinite(sel->expand) && sel->expand >= 0.0f, "%s: expand %g; a finite value >= 0 is required", api, (double) sel->expand);
    if (int rc = snn::checkDevicePointer(api, rows, sizeof(float), ctx->device, "rows", 0)) return rc;
    if (int rc = snn::checkDevicePointer(api, counts, sizeof(int), ctx->device, "counts", 0)) return rc;
    if (int rc = snn::checkDevicePointer(api, rois, sizeof(int), ctx->device, "rois", 0)) return rc;
    if (int rc = snn::checkDevicePointer(api, count, sizeof(int), ctx->device, "count", 0)) return rc;
    if (int rc = snn::checkCallerStream(api, stream)) return rc;
    if (frameWh)
        return snnb::launch_rois_from_detections(ctx, stream ? stream : ctx->stream, rows, counts, numFrames, maxRows, frameWh, *sel, rois, capacity, count);
    return snnb::launch_rois_from_detections(ctx, stream ? stream : ctx->stream, rows, counts, numFrames, maxRows, fw, fh, *sel, rois, capacity, count);
}
int snnb::rois_from_detections(snnb_context* ctx, const float* rows, const int* counts, int numFrames, int maxRows, int fw, int fh, const snnb_roi_select* sel,
                               snnb_roi* rois, int capacity, int* count, cudaStream_t stream) {
    return roisFromDetections("snnb_rois_from_detections", ctx, rows, counts, numFrames, maxRows, fw, fh, nullptr, sel, rois, capacity, count, stream);
}
int snnb::rois_from_detections_list(snnb_context* ctx, const float* rows, const int* counts, int numFrames, int maxRows, const int* frameWh,
                                    const snnb_roi_select* sel, snnb_roi* rois, int capacity, int* count, cudaStream_t stream) {
    SNNB_REQUIRE(frameWh, "snnb_rois_from_detections_list: null frame_wh");
    return roisFromDetections("snnb_rois_from_detections_list", ctx, rows, counts, numFrames, maxRows, 0, 0, frameWh, sel, rois, capacity, count, stream);
}
