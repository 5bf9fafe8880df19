"""CPU checks of what test_converted_exact_gpu.py runs: oracle/exact.py's restatements of converted layers against the source's own
float64 semantics, independent of the engine.

- Coverage: every branch and attribute form of onnx2snn.convert_graph is reached by the GPU table's graphs, read from the layers the
  converter writes for them.
- Semantics: each converted layer, restated in float64 from the source's float64 values of its inputs (onnx2snn.torch_eval), lies within
  the restatement's bound of the source's value of the tensor it stands for; the exports' restated layer chain ends within the bound of
  the torchvision module's float64 logits. This pins the oracle's (and so the engine's) reading of every converted attribute to ONNX /
  torch semantics.
- Mutations: plausible misreadings of a converted attribute land outside the bound somewhere in the same data.
- Refusals: the forms the engine has no counterpart for are refused with a ValueError naming the attribute.
"""
import os

import numpy as np
import pytest

from oracle import exact, oracle
from shadernn_b200 import modelzoo, onnx2snn

import _converted_graphs as cg
from _candy_fixture import head_graph
import test_layer_exact_gpu as tl

pytestmark = pytest.mark.usefixtures("built")

SIMT = "conv2d_simt"  # restate every convolution as the CUDA-core kernel does: the plainest fp32 statement


def nhwc(t):
    return t.permute(0, 2, 3, 1).contiguous().numpy()


def cases():
    """(label, graph dict, input) of every graph-dict and Candy case the GPU table converts with fold_pads=True."""
    out = [("graph " + k, f(), cg.graph_input(k)) for k, f in sorted(cg.GRAPHS.items())]
    g, x, _ = head_graph()
    out.append(("candy head 64x64", g, x.astype(np.float64)))
    out.append(("candy head 70x131", head_graph()[0], cg.candy_input(2, 70, 131, seed=70)))
    return out


def layer_semantics(tmp, label, g, x, layers=None):
    """Worst |restatement - source| / bound over every converted layer, and the number of elements outside."""
    import torch
    if layers is None:
        layers = onnx2snn.convert_graph(g, input_hw=x.shape[1:3])
    path = modelzoo.write_model(layers, os.path.join(tmp, label.replace(" ", "_") + "_layers.json"), split=True)
    om = oracle.Model(path)
    vals = onnx2snn.torch_eval(g, x, dtype=torch.float64, return_all=True)
    # every layer's inputs as an fp32 tensor holds them, as the restatements take their operands
    outs = [exact.stored(nhwc(vals[l["_onnx"]]), False) for l in layers]
    kernels = {"names": [SIMT] * len(layers), "shapes": [o.shape for o in outs]}
    producer = {}
    for nd in g["nodes"]:
        producer[nd["output"][0]] = nd
    worst, bad = 0.0, 0
    for i in range(1, len(layers)):
        l = layers[i]
        ins = [layers[int(j)]["_onnx"] for j in l["inputId"]]
        # the source nodes this layer stands for, evaluated in float64 from the same fp32 inputs
        sub, todo = [], [l["_onnx"]]
        while todo:
            t = todo.pop()
            if t in ins or t not in producer or producer[t] in sub:
                continue
            sub.append(producer[t])
            todo += [u for u in producer[t]["input"] if u and u not in g["init"]]
        sub = [nd for nd in g["nodes"] if nd in sub]
        want = nhwc(onnx2snn.torch_eval(dict(g, nodes=sub), None, dtype=torch.float64, return_all=True,
                                        feeds={t: outs[int(j)] for t, j in zip(ins, l["inputId"])})[l["_onnx"]])
        r = tl.restate(om, i, outs, kernels, "fp32x3", False, x)
        assert r is not None, (label, i, l["type"])
        ref, bound = r
        assert ref.shape == want.shape, (label, i, ref.shape, want.shape)
        ratio, b = exact.check(want, ref, bound, l["type"])
        worst, bad = max(worst, ratio), bad + b
    return worst, bad


@pytest.mark.parametrize("case", range(5), ids=["depthwise_bn", "pads", "resize", "candy64", "candy70x131"])
def test_restatements_agree_with_source(tmp_path, case):
    label, g, x = cases()[case]
    worst, bad = layer_semantics(str(tmp_path), label, g, x)
    print("%-20s worst |restated - source| / bound %.3g" % (label, worst))
    assert bad == 0, (label, worst)


@pytest.mark.parametrize("name", ["resnet18", "mobilenet_v2"])
def test_export_restatements_agree_with_torch(tmp_path, name):
    import torch
    import torchvision
    from shadernn_b200 import convert
    torch.manual_seed(11)
    model = getattr(torchvision.models, name)(weights=None, num_classes=37)
    gen = torch.Generator().manual_seed(12)
    for m in model.modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            m.weight.data.uniform_(0.5, 1.5, generator=gen)
            m.bias.data.uniform_(-0.1, 0.1, generator=gen)
            m.running_mean.uniform_(-0.1, 0.1, generator=gen)
            m.running_var.uniform_(0.5, 1.5, generator=gen)
    model.eval()
    hw = (64, 64)
    path = str(tmp_path / (name + ".json"))
    convert.export(model, path, input_hw=hw, split=True)
    x = np.random.default_rng(4).uniform(-1, 1, (2,) + hw + (3,))
    om = oracle.Model(path)
    shapes = [o.shape for o in om.run(x.astype(np.float32), return_all=True)]
    outs = [None] * om.count
    kernels = {"names": [SIMT] * om.count, "shapes": shapes}
    for i in range(om.count):
        ref, bound = tl.restate(om, i, outs, kernels, "fp32x3", False, x)
        outs[i] = ref
    with torch.no_grad():
        want = model.double()(torch.from_numpy(x).permute(0, 3, 1, 2)).numpy()
    ratio, bad = exact.check(want.reshape(ref.shape), ref, bound, "logits")
    print("%-14s restated chain vs torch float64 logits: |err| / last layer's bound %.3g" % (name, ratio))
    assert bad == 0


def conv_forms(layers, g):
    """The convert_graph forms a converted model reaches, as tags."""
    tags = set()
    ops = {nd["output"][0]: nd for nd in g["nodes"]}
    for l in layers:
        t = l["type"]
        if t in ("Conv2D", "DepthwiseConv2D"):
            k, s = int(l["kernel_size"]), int(l["strides"])
            p = l["padding"]
            tags |= {(t, "k", k), (t, "stride", s), (t, "bias", l["useBias"]), (t, "bn", l["useBatchNormalization"]), (t, "act", l["activation"])}
            if isinstance(p, list):
                tags.add((t, "pads", "symmetric" if p[0][0] == p[0][1] else "asymmetric"))
                tags.add((t, "mode", l.get("mode", "constant")))
            else:
                tags.add((t, "pads", p))
        elif t == "Pad":
            pd = l["pads"]
            tags.add(("Pad", "standalone", l["mode"], "symmetric" if pd[2] == pd[6] and pd[3] == pd[7] else "asymmetric"))
        elif t == "UpSampling2D":
            nd = ops[l["_onnx"]] if l["_onnx"] in ops else None
            tags.add(("UpSampling2D", l["interpolation"], float(l["scaleFactor"]), nd["op"] if nd else "",
                      nd["attr"].get("coordinate_transformation_mode", "") if nd else ""))
        elif t in ("Activation", "BatchNormalization", "Add", "InstanceNormalization", "MaxPooling2D", "AveragePooling2D", "Concatenate"):
            tags.add((t, l.get("activation", "")))
        if l.get("activation", "linear") != "linear":
            tags.add(("activation", l["activation"], "standalone" if t == "Activation" else "fused"))
    for nd in g["nodes"]:
        if nd["op"] == "Pad" and nd["output"][0] not in {l.get("_onnx") for l in layers}:
            p = nd["attr"]["pads"]
            tags.add(("Pad", "folded", onnx2snn._PAD_MODE[nd["attr"]["mode"]], "symmetric" if p[2] == p[6] else "asymmetric"))
        if nd["op"] == "BatchNormalization":
            standalone = nd["output"][0] in {l.get("_onnx") for l in layers if l["type"] == "BatchNormalization"}
            tags.add(("BatchNormalization", "standalone" if standalone else "folded", float(np.float32(nd["attr"]["epsilon"]))))
        if nd["op"] in ("Upsample", "Resize"):
            sc = float(g["init"][nd["input"][-1]].ravel()[2])
            tags.add((nd["op"], nd["attr"]["mode"], sc, nd["attr"].get("coordinate_transformation_mode", "half_pixel" if nd["op"] == "Resize" else "")))
    return tags


def test_gpu_table_reaches_every_converter_form():
    tags = set()
    for fold in (True, False):
        g = head_graph()[0]
        tags |= conv_forms(onnx2snn.convert_graph(g, input_hw=(64, 64), fold_pads=fold), g)
    for f in cg.GRAPHS.values():
        g = f()
        tags |= conv_forms(onnx2snn.convert_graph(g), g)
    want = set()
    for mode in ("constant", "reflect", "replicate"):
        want |= {("Pad", "folded", mode, "symmetric"), ("Pad", "standalone", mode, "symmetric" if mode != "replicate" else "asymmetric")}
    want |= {("Pad", "folded", "constant", "asymmetric"), ("Pad", "folded", "replicate", "symmetric")}
    want |= {("Conv2D", "k", k) for k in (1, 2, 3, 5, 9)} | {("Conv2D", "stride", s) for s in (1, 2)}
    want |= {("Conv2D", "pads", p) for p in ("symmetric", "asymmetric", "valid")} | {("Conv2D", "bias", b) for b in ("True", "False")}
    want |= {("Conv2D", "mode", m) for m in ("constant", "reflect", "replicate")}
    want |= {("DepthwiseConv2D", "stride", s) for s in (1, 2)} | {("DepthwiseConv2D", "bn", "True"), ("DepthwiseConv2D", "act", "relu6")}
    want |= {("BatchNormalization", how, float(np.float32(e))) for how in ("folded", "standalone") for e in (1e-5, 1e-3)}
    want |= {("activation", a, how) for a in ("relu", "relu6", "leakyRelu", "tanh", "sigmoid") for how in ("fused", "standalone")}
    want |= {("InstanceNormalization", "linear"), ("InstanceNormalization", "relu"), ("Add", "linear"), ("Add", "relu"), ("Concatenate", "")}
    want |= {("MaxPooling2D", ""), ("AveragePooling2D", "")}
    want |= {("Resize", "nearest", 2.0, "half_pixel"), ("Resize", "nearest", 2.0, "asymmetric"), ("Upsample", "nearest", 2.0, "")}
    want |= {("Resize", "linear", 2.0, m) for m in ("half_pixel", "pytorch_half_pixel")} | {("Resize", "linear", 1.5, "half_pixel")}
    want |= {("Resize", "linear", 1.0, m) for m in ("half_pixel", "asymmetric", "align_corners")}
    missing = sorted(map(str, want - tags))
    assert not missing, missing


@pytest.mark.parametrize("case", sorted(cg.REFUSED))
def test_converter_refuses(case):
    make, attribute = cg.REFUSED[case]
    with pytest.raises(ValueError, match=attribute):
        onnx2snn.convert_graph(make())


# ---- mutations: each misreading must leave the bound somewhere in the GPU table's data -----------------------------------------
def mutated_layers(g, how):
    layers = onnx2snn.convert_graph(g)
    for l in layers:
        if how == "pads begin and end swapped" and isinstance(l.get("padding"), list):
            (t, b), (lft, r) = l["padding"]
            l["padding"] = [[b, t], [r, lft]]
        if how == "pads begin and end swapped" and l["type"] == "Pad":
            p = l["pads"]
            l["pads"] = [0, 0, p[6], p[7], 0, 0, p[2], p[3]]
        if how == "edge as zero padding" and l.get("mode") == "replicate":
            l["mode"] = "constant"
        if how == "depthwise kernel transposed" and l["type"] == "DepthwiseConv2D":
            l["_w"]["kernel_chw"] = l["_w"]["kernel_chw"].transpose(0, 2, 1).copy()
    return layers


def _bn_fold_wrong_way(bn, eps):
    var = bn["moving_variance"].astype(np.float64)
    bn["gamma"] = (bn["gamma"] * np.sqrt(var + float(np.float32(eps))) / np.sqrt(var + 1e-3)).astype(np.float32)
    return bn


def _half_pixel_dropped(real):
    def coord(o, size, scale):
        _, e = real(o, size, scale)
        return np.clip(np.asarray(o, np.float64) / float(np.float32(scale)), 0, size - 1), e
    return coord


MUTATIONS = ["pads begin and end swapped", "edge as zero padding", "depthwise kernel transposed", "BN epsilon folded the wrong way",
             "bilinear without the half-pixel offset", "InstanceNorm epsilon 1e-3"]


@pytest.mark.parametrize("how", MUTATIONS)
def test_mutations_leave_the_bound(tmp_path, monkeypatch, how):
    if how == "BN epsilon folded the wrong way":
        monkeypatch.setattr(onnx2snn, "_bn_fold_eps", _bn_fold_wrong_way)
    if how == "bilinear without the half-pixel offset":
        monkeypatch.setattr(exact, "bilinear_coord", _half_pixel_dropped(exact.bilinear_coord))
    if how == "InstanceNorm epsilon 1e-3":
        real = exact.instancenorm
        monkeypatch.setattr(exact, "instancenorm", lambda *a, **k: real(*a, **dict(k, eps=1e-3)))
    hit = []
    for label, g, x in cases():
        layers = mutated_layers(g, how)
        worst, bad = layer_semantics(str(tmp_path), label, g, x, layers)
        if bad:
            hit.append((label, worst))
    print("%-40s caught in %s" % (how, hit))
    assert hit, how

