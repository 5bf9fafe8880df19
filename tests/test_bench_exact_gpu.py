"""The benchmark's own batches held to the layer-local float64 bounds of oracle/exact.py, on every image.

test_layer_exact_gpu.py restates whole layers at small shapes. The configurations bench.py times are larger: the planner picks wide
tiles there, stacks images in one tile box and runs several waves of the persistent loop, and those are the launches a defect in
a later wave, a later image or a tile box's image boundary would show in. Restating these batches whole in float64 takes too long,
so each layer is restated at chosen output pixels (exact.sample_pixels), for all channels:

- every pixel of the first and last output row and column of every image (padding, tile overhang at the right and bottom edges);
- a convolution: two seeded random pixels in every tile of its launch, the tile boxes taken from the plan the engine launched
  (test_conv_plan.plan = snnb_debug_conv_launch at the layer's query, batch and precision, checked against the kernel each layer
  ran). With all channels checked at each pixel, every channel tile, every K piece and every wave has checked outputs;
- every other layer: one seeded random pixel in every 8 x 8 block of each image.

Layers that only move data (input upload, pad, concat, flatten, nearest upsampling), the classifier heads and all of ESPCN are
restated whole. The pixels depend only on (model, layer, SEED), so a failure reproduces.

Each case runs the model as bench.py's Workload does: modelzoo.build at the model's default size, fused, through a CUDA graph,
the default convolution algorithm, bench.py's synthetic input for the rank. The checked replay follows passes on bench.py's other
input, so no tensor already holds the value the replay is to give it.
"""
import time
import zlib

import numpy as np
import pytest

from oracle import exact, oracle
from shadernn_b200 import core, modelzoo

pytestmark = pytest.mark.gpu

FORMS = ("fp32x3", "fp16w", "fp16")
SEED = 0
WORLD = 8  # the strong-scaling runs of BASELINE.json configs[2..4] shard the bench batch over 8 ranks
STRONG = ("mobilenetv2", "yolov3tiny", "candy")
WHOLE_MODELS = ("espcn",)  # cheap enough to restate in full
DATA_MOVES = ("InputLayer", "Pad", "Concatenate", "Flatten", "UpSampling2D")  # bound 0: compared in full, bit for bit
PATH_KERNEL = {2: "conv_umma_kernel", 3: "conv_rowwin_kernel", 4: "conv_rowwin_kernel<feed>"}  # test_conv_plan IGEMM, ROWWIN, FEED


def bench_cases():
    """(model, batch, precision, rank): every bench.WORKLOADS entry in every precision at rank 0, and the last rank's shard of each
    strong-scaling run in fp32x3."""
    import bench
    from shadernn_b200 import parallel
    cases = [(key, batch, precision, 0) for key, batch, _ in bench.WORKLOADS.values() for precision in FORMS]
    for key in STRONG:
        batch = bench.WORKLOADS[key][1]
        _, count = parallel.shard_range(batch, WORLD, WORLD - 1)
        cases.append((key, count, "fp32x3", WORLD - 1))
    return cases


def inputs_of(l):
    return [int(v) for v in l.get("inputId", [])][:int(l.get("numInputs", 0))]


def fused_convs(om):
    """The engine's fusion of each Conv2D of oracle.Model om (MixedInferenceCore::init, fuse on): {conv: (source layer whose tensor it
    reads, folded Pad layer or None, the Add whose epilogue it runs or None)}."""
    consumers = {}
    for i, l in enumerate(om.layers):
        for j in inputs_of(l):
            consumers.setdefault(j, []).append(i)
    order, pending, ready = {}, [i for i, l in enumerate(om.layers) if not inputs_of(l)], {}
    while pending:  # the engine's execution order: Kahn's algorithm, ready layers taken in JSON order (dp.cpp)
        i = pending.pop(0)
        order[i] = len(order)
        for q in consumers.get(i, []):
            ready[q] = ready.get(q, 0) + 1
            if ready[q] == len(inputs_of(om.layers[q])):
                pending.append(q)
    out, adds = {}, {}
    for j, l in enumerate(om.layers):
        if om.type_of(l) != "Conv2D":
            continue
        k = int(l["kernel_size"])
        src, pad = inputs_of(l)[0], None
        p = om.layers[src]
        if (om.type_of(p) == "Pad" and k > 1 and len(consumers.get(src, [])) == 1 and len(inputs_of(p)) == 1
                and om._offsets(l, k) == [0, 0, 0, 0]):
            src, pad = inputs_of(p)[0], src
        cons = consumers.get(j, [])
        if l.get("activation", "linear") in ("", "linear") and len(cons) == 1 and om.type_of(om.layers[cons[0]]) == "Add":
            ins = inputs_of(om.layers[cons[0]])
            if len(ins) == 2 and j in ins:
                adds.setdefault(cons[0], []).append(j)
        out[j] = [src, pad, None]
    for a, convs in adds.items():  # the second operand first, as the fusion pass tries it; the other operand must run earlier
        ins = inputs_of(om.layers[a])
        for c in sorted(convs, key=lambda c: -ins.index(c)):
            other = ins[1 - ins.index(c)]
            if order[other] < order[c]:
                out[c][2] = a
                break
    return {j: tuple(v) for j, v in out.items()}


def conv_query(om, j, fusion, shapes):
    """test_conv_plan.plan's arguments for Conv2D j as the engine plans it (Conv2DLayer::plan), from the per-layer NHWC shapes."""
    import test_conv_plan as cp
    l = om.layers[j]
    k, s = int(l["kernel_size"]), int(l["strides"])
    src, pad, add = fusion[j]
    spec = om.layers[pad] if pad is not None else l
    o = om._offsets(spec, 0, False) if pad is not None else om._offsets(l, k)
    mode = spec.get("mode", "constant") if pad is not None else (l.get("mode", "constant") if "mode" in l else "")
    pad_mode = {"": cp.PAD_NONE, "constant": cp.PAD_CONSTANT, "replicate": cp.PAD_REPLICATE, "reflect": cp.PAD_REFLECT}[mode]
    first = min(q for q in fusion if om.type_of(om.layers[fusion[q][0]]) == "InputLayer") if any(
        om.type_of(om.layers[fusion[q][0]]) == "InputLayer" for q in fusion) else None
    return dict(in_hwc=tuple(shapes[src][1:]), out_hwc=tuple(shapes[j][1:]), k=k, stride=s, pad_x=0 if k == 1 else o[0],
                pad_y=0 if k == 1 else o[2], pad_mode=pad_mode, residual=add is not None, may_feed=j == first)


def conv_plan(query, n, precision, sms):
    import test_conv_plan as cp
    q = dict(query)
    return cp.plan(q.pop("in_hwc"), q.pop("out_hwc"), q.pop("k"), q.pop("stride"), q.pop("pad_x"), q.pop("pad_y"), n=n, precision=precision,
                   sms=sms, **q)


def plan_kernel(p):
    """The name MixedInferenceCore.layer_kernel reports for a launch of plan p."""
    name = PATH_KERNEL.get(p["path"], "conv2d_simt_kernel")
    if p["path"] == 2 and (p["sk"] or p["ksplit"] > 1):
        name += "<stream-K>" if p["sk"] else "<split-K>"
    return name


def tile_box(p):
    """The output box of one tile of plan p: (tw, th, tn). conv_umma_kernel's tile is the plan's box on its tiles_x x tiles_y x tiles_n
    grid; conv_rowwin_kernel's is 128 pixels of one output row of one image (its tmO box, UM_BLOCK_M x 1 x 1, tile = (n, oy, xt))."""
    if p["path"] == 2:
        return (p["tw"], p["th"], p["tn"])
    if p["path"] in (3, 4):
        return (128, 1, 1)
    return None


def layer_seed(key, i):
    return [zlib.crc32(key.encode()), i, SEED]


def choose_pixels(key, i, shape, box):
    """Output pixels of layer i (NHWC shape): the edges, plus two per tile of `box` for a convolution, one per 8 x 8 block otherwise."""
    n, oh, ow, _ = shape
    if box is not None:
        return exact.sample_pixels(n, oh, ow, [box], layer_seed(key, i), per_box=2)
    return exact.sample_pixels(n, oh, ow, [(8, 8, 1)], layer_seed(key, i), per_box=1)


def last_uses(om):
    """For each layer, the last layer whose restatement may read its output: restate() reads past a folded Pad, a fused Flatten or
    average pool and a Conv2D fused into its Add, so their inputs are kept as long as their consumers."""
    last = list(range(om.count))

    def reads(i, seen):
        for j in inputs_of(om.layers[i]):
            if j not in seen:
                seen.add(j)
                if om.type_of(om.layers[j]) in ("Pad", "Flatten", "AveragePooling2D", "Conv2D"):
                    reads(j, seen)
        return seen

    for i in range(om.count):
        for j in reads(i, set()):
            last[j] = max(last[j], i)
    return last


def run_case(ctx, model_dir, key, batch, precision, rank):
    import test_layer_exact_gpu as tl
    import torch
    from shadernn_b200._lib import SnnbError
    sms = torch.cuda.get_device_properties(ctx.device).multi_processor_count
    path, _ = modelzoo.build(key, model_dir)
    x = modelzoo.synthetic_input(key, batch, seed=7767517 + rank)
    om = oracle.Model(path)
    half = precision == "fp16"
    m = core.MixedInferenceCore(ctx, path, batch=batch, use_cuda_graph=True, fuse=True, precision=precision)
    checked, pixels, worst, skipped, cpu = 0, 0, 0.0, [], 0.0
    try:
        # Warm-up and the eager pass that names each layer's kernel run on bench.py's other input (its second buffer), so that every
        # tensor holds another image's values when the checked replay starts: a read that comes too early in that replay (a missing
        # dependency, a residual or activation fetched before its producer finished) sees stale values and fails the bounds
        m.set_input(modelzoo.synthetic_input(key, batch, seed=99 + rank))
        m.forward()
        ctx.sync()
        m.time_layers()
        kernels = {"names": [m.layer_kernel(i) for i in range(m.num_layers)], "shapes": [m.layer_info(i)[2] for i in range(m.num_layers)]}
        m.set_input(x)
        m.forward()  # the graph replay whose outputs are checked
        ctx.sync()
        fusion = fused_convs(om)
        boxes = {}
        for j in fusion:
            p = conv_plan(conv_query(om, j, fusion, kernels["shapes"]), batch, precision, sms)
            assert kernels["names"][j] == plan_kernel(p), (key, precision, j, kernels["names"][j], p)
            boxes[j] = tile_box(p)
            if fusion[j][2] is not None:
                boxes[fusion[j][2]] = boxes[j]
        last = last_uses(om)
        outs = [None] * om.count
        for i in range(om.count):
            t = om.type_of(om.layers[i])
            if t != "YOLO" and not (t in ("Pad", "Flatten") and kernels["names"][i] == ""):  # a folded Pad or fused Flatten has no tensor
                try:
                    outs[i] = m.layer_output(i)
                except SnnbError:
                    assert i in fusion and fusion[i][2] is not None or t == "AveragePooling2D", m.layer_info(i)
            if i in fusion:
                assert (outs[i] is None) == (fusion[i][2] is not None), ("conv fused into its Add", i, fusion[i])
            if outs[i] is not None:
                t0 = time.perf_counter()
                n, oh, ow, _ = outs[i].shape
                if t in ("Dense", "Softmax"):
                    parts = [None]  # the classifier heads, restated whole
                elif key in WHOLE_MODELS or t in DATA_MOVES:
                    # every pixel, one image at a time: a whole 720 x 720 x 64 batch in float64 with its temporaries would take gigabytes
                    parts = [(np.full(oh * ow, q), *np.indices((oh, ow)).reshape(2, -1)) for q in range(n)]
                else:
                    parts = [choose_pixels(key, i, outs[i].shape, boxes.get(i))]
                for at in parts:
                    r = tl.restate(om, i, outs, kernels, precision, half, x, at)
                    if r is None:
                        skipped.append("%d:%s" % (i, t))
                        break
                    ref, bound = r
                    got = outs[i] if at is None else outs[i][at]
                    assert got.shape == ref.shape, (key, i, t, got.shape, ref.shape)
                    ratio, bad = exact.check(got, ref, bound, t)
                    assert bad == 0, "%s batch %d %s rank %d: layer %d (%s, %s): %d of %d values outside the bound, worst |err|/bound %.3g" % (
                        key, batch, precision, rank, i, t, kernels["names"][i], bad, ref.size, ratio)
                    worst = max(worst, ratio)
                    pixels += ref.size // ref.shape[-1]
                checked += r is not None
                cpu += time.perf_counter() - t0
            for j in range(i + 1):
                if last[j] <= i:
                    outs[j] = None
    finally:
        m.close()
    print("%-12s batch %2d %-6s rank %d: %3d layers, %8d pixels restated, worst |err|/bound %.3g, %.1f s restating%s" % (
        key, batch, precision, rank, checked, pixels, worst, cpu, (" (not restated: %s)" % ", ".join(skipped)) if skipped else ""))
    assert not skipped, "layers without a restatement: %s" % skipped
    return worst


CASES = bench_cases()


@pytest.mark.parametrize("key,batch,precision,rank", CASES, ids=["%s-n%d-%s-r%d" % c for c in CASES])
def test_bench_batch_layer_exact(ctx, model_dir, key, batch, precision, rank):
    run_case(ctx, model_dir, key, batch, precision, rank)
