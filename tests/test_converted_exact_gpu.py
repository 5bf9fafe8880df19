"""Layer-local, teacher-forced checks of converted models: every layer of a model written by shadernn_b200/onnx2snn.convert_graph or
shadernn_b200/convert.export held to oracle/exact.py's float64 restatement fed the engine's own inputs (test_layer_exact_gpu.py's walker),
in fp32x3, fp16w and fp16, fused and unfused, on the tensor-core and the CUDA-core convolutions.

- The real-weight Candy head (tests/golden/candy_head_golden.npz) with its reflect Pads folded into the convolutions and kept standalone,
  at 64x64 and 70x131 (odd sides, two images), on 0..255 input; the 9x9 stem's kernel is asserted.
- torchvision ResNet-18 and MobileNetV2 through convert.export, with randomised BatchNorm statistics.
- Graph dicts built in tests/_converted_graphs.py that reach every branch of convert_graph. For these the engine's shape of every layer
  must also be the source graph's shape of the tensor the layer stands for.
"""
import os

import numpy as np
import pytest

from shadernn_b200 import convert, modelzoo, onnx2snn

import _converted_graphs as cg
from _candy_fixture import head_graph
from test_layer_exact_gpu import FORMS, teacher_forced_model

pytestmark = pytest.mark.gpu

ALGOS = ("auto", "simt")


def source_shapes(g, x, layers):
    import torch
    vals = onnx2snn.torch_eval(g, x, dtype=torch.float64, return_all=True)
    return {i: tuple(int(d) for d in vals[l["_onnx"]].permute(0, 2, 3, 1).shape) for i, l in enumerate(layers) if "_onnx" in l}


def run_graph(ctx, tmp, label, g, x, fold, precision, fuse, algo, check_shapes):
    n, h, w, _ = x.shape
    layers = onnx2snn.convert_graph(g, input_hw=(h, w), fold_pads=fold)
    path = modelzoo.write_model(layers, os.path.join(tmp, "%s_%d_layers.json" % (label.replace(" ", "_"), int(fold))), split=True)
    _, _, kernels = teacher_forced_model(ctx, path, x, n, (h, w), precision, fuse, algo, label=label)
    if check_shapes:
        for i, want in source_shapes(g, x, layers).items():
            if i == 0:
                continue
            assert kernels["shapes"][i] == want, (label, i, layers[i]["type"], kernels["shapes"][i], want)
    return layers, kernels


@pytest.mark.parametrize("algo", ALGOS)
@pytest.mark.parametrize("fuse", [False, True])
@pytest.mark.parametrize("precision", FORMS)
def test_real_candy_head(ctx, tmp_path, precision, fuse, algo):
    g, x64, _ = head_graph()
    for fold, (h, w), n in cg.CANDY:
        x = x64 if (h, w, n) == (64, 64, 1) else cg.candy_input(n, h, w, seed=h)
        label = "candy head %s %dx%d" % ("folded" if fold else "pads", h, w)
        # fold_pads=False keeps the reference tool's literal layout (an unpadded convolution keeps its input's size): no source shapes
        layers, kernels = run_graph(ctx, str(tmp_path), label, g, x, fold, precision, fuse, algo, check_shapes=fold)
        stem = [i for i, l in enumerate(layers) if l["type"] == "Conv2D"][0]
        name = kernels["names"][stem]
        if algo == "simt":
            assert name.startswith("conv2d_simt"), (label, name)
        else:  # 3 input channels, stride 1: the small-channel row-window kernel
            assert name.startswith("conv_rowwin_kernel"), (label, name)


@pytest.mark.parametrize("name", ["resnet18", "mobilenet_v2"])
@pytest.mark.parametrize("precision", FORMS)
def test_torchvision_exports(ctx, tmp_path, name, precision):
    import torch
    import torchvision
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
    # the exporter writes the global pool as a square pool of H / 32: sizes are square multiples of 32. The second size runs fused on
    # the tensor cores only, to keep the file's time down
    for hw, n, runs in (((96, 96), 5, ((False, "auto"), (True, "auto"), (False, "simt"), (True, "simt"))), ((160, 160), 1, ((True, "auto"),))):
        path = str(tmp_path / ("%s_%d.json" % (name, hw[0])))
        convert.export(model, path, input_hw=hw, split=True)
        x = np.random.default_rng(hw[0]).uniform(-1, 1, (n,) + hw + (3,)).astype(np.float32)
        for fuse, algo in runs:
            teacher_forced_model(ctx, path, x, n, hw, precision, fuse, algo, label=name)


@pytest.mark.parametrize("algo", ALGOS)
@pytest.mark.parametrize("fuse", [False, True])
@pytest.mark.parametrize("precision", FORMS)
@pytest.mark.parametrize("graph", sorted(cg.GRAPHS))
def test_graph_dicts(ctx, tmp_path, graph, precision, fuse, algo):
    g = cg.GRAPHS[graph]()
    run_graph(ctx, str(tmp_path), "graph " + graph, g, cg.graph_input(graph), True, precision, fuse, algo, check_shapes=True)

