"""Generator of tests/golden/candy_head_golden.npz — run where a checkout of the reference exists:

    python tests/golden/make_candy_golden.py <reference checkout>/modelzoo/StyleTransfer/candy-9_simplified.onnx

The only real-weight model in the reference checkout is modelzoo/StyleTransfer/candy-9_simplified.onnx. At 6.7 MB it is not
part of this repository, so this script freezes (a) the initialisers of its first two stages (reflect-pad + 9x9 conv 3->32 + InstanceNorm +
ReLU; reflect-pad + 3x3 stride-2 conv 32->64 + InstanceNorm + ReLU: ~105 KB of fp32), (b) a 64x64 input in the model's own
range [0, 255], and (c) what torch computes for those ONNX nodes (shadernn_b200/onnx2snn.torch_eval on the truncated graph,
i.e. the ONNX semantics themselves, no conversion involved). tests/ rebuild the SNN model from (a) with the converter and
hold the oracle and the CUDA engine to (c). With SNNB_REFERENCE set to a reference checkout, __graft_entry__.build() also converts
the WHOLE model into tests/golden/_ref_models/ (git-ignored) with a full-size golden output beside it (full_model below).
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from shadernn_b200 import modelzoo, onnx2snn  # noqa: E402

HEAD_NODES = 8  # Pad Conv IN Relu Pad Conv IN Relu


def truncated(g, n_nodes):
    nodes = g["nodes"][:n_nodes]
    used = {t for nd in nodes for t in nd["input"]}
    return {"nodes": nodes, "init": {k: v for k, v in g["init"].items() if k in used}, "inputs": g["inputs"], "outputs": [(nodes[-1]["output"][0], [])]}


def main(src):
    g = onnx2snn.load_onnx(src)
    head = truncated(g, HEAD_NODES)
    x = modelzoo.synthetic_input("candy", 1, (64, 64))
    y = onnx2snn.torch_eval(head, x)
    out = {"x": x, "y": y, "node_ops": np.array([nd["op"] for nd in head["nodes"]])}
    for k, v in head["init"].items():
        out["init/" + k] = np.array(v)
    path = os.path.join(ROOT, "tests", "golden", "candy_head_golden.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes; output", y.shape, "max", float(np.abs(y).max()))


def full_model(src, out_dir, hw=(224, 224)):
    """Whole-model conversion + golden output (torch on the ONNX graph) for the GPU tests; returns the JSON path."""
    os.makedirs(out_dir, exist_ok=True)
    g = onnx2snn.load_onnx(src)
    path, _ = onnx2snn.convert(src, out_dir, input_hw=hw)
    x = modelzoo.synthetic_input("candy", 1, hw)
    np.savez_compressed(os.path.join(out_dir, "candy_full_golden.npz"), x=x, y=onnx2snn.torch_eval(g, x))
    return path


if __name__ == "__main__":
    main(sys.argv[1])
