"""ONNX graph dicts (shadernn_b200/onnx2snn.load_onnx's form) that between them reach every branch and attribute form of
convert_graph: the cases of test_converted_exact_gpu.py and test_converted_exact_cpu.py, and the forms the converter refuses."""
import numpy as np


class Graph:
    """A graph dict under construction: seeded He-normal weights, node outputs named after the nodes."""

    def __init__(self, name, c, h, w, seed):
        self.rng = np.random.default_rng(seed)
        self.name = name
        self.g = {"nodes": [], "init": {}, "inputs": [("x", [1, c, h, w])], "outputs": []}
        self.planes = {"x": c}

    def node(self, op, ins, attr=None, planes=None):
        out = "%s%d" % (op.lower(), len(self.g["nodes"]))
        self.g["nodes"].append({"op": op, "input": list(ins), "output": [out], "name": out, "attr": dict(attr or {})})
        self.planes[out] = planes if planes is not None else self.planes[ins[0]]
        return out

    def const(self, name, a):
        self.g["init"][name] = np.asarray(a, np.float32)
        return name

    def conv(self, x, oc, k, s=1, pads=(0, 0, 0, 0), bias=True, group=1, gain=1.0):
        ic = self.planes[x] // group
        w = self.const("w%d" % len(self.g["nodes"]), self.rng.standard_normal((oc, ic, k, k)) * np.sqrt(2.0 / (ic * k * k)) * gain)
        ins = [x, w] + ([self.const("b%d" % len(self.g["nodes"]), self.rng.uniform(-0.1, 0.1, oc))] if bias else [])
        return self.node("Conv", ins, {"kernel_shape": [k, k], "strides": [s, s], "pads": list(pads), "group": group}, planes=oc)

    def pad(self, x, t, b, l, r, mode="constant"):  # ONNX order: x1_begin .. x4_begin, x1_end .. x4_end
        return self.node("Pad", [x], {"mode": mode, "pads": [0, 0, t, l, 0, 0, b, r]})

    def bn(self, x, eps):
        c, n = self.planes[x], len(self.g["nodes"])
        ins = [x] + [self.const("bn%d_%s" % (n, k), v) for k, v in (("g", self.rng.uniform(0.5, 1.5, c)), ("b", self.rng.uniform(-0.2, 0.2, c)),
                                                                  ("m", self.rng.uniform(-0.2, 0.2, c)), ("v", self.rng.uniform(0.5, 1.5, c)))]
        ins[4] = self.const("bn%d_v" % n, np.exp(self.rng.uniform(np.log(1e-4), np.log(2.0), c)))  # small variances too: where eps matters
        return self.node("BatchNormalization", ins, {"epsilon": eps})

    def instance_norm(self, x, eps=1e-5):
        c, n = self.planes[x], len(self.g["nodes"])
        return self.node("InstanceNormalization", [x, self.const("in%d_g" % n, self.rng.uniform(0.5, 1.5, c)), self.const("in%d_b" % n, self.rng.uniform(-0.2, 0.2, c))],
                         {"epsilon": eps})

    def resize(self, x, scale, mode, ctm=None, nearest_mode=None, op="Resize"):
        n = len(self.g["nodes"])
        a = {"mode": mode}
        if ctm:
            a["coordinate_transformation_mode"] = ctm
        if nearest_mode:
            a["nearest_mode"] = nearest_mode
        sc = self.const("sc%d" % n, [1, 1, scale, scale])
        return self.node(op, [x, "", sc] if op == "Resize" else [x, sc], a)

    def clip(self, x, lo=0.0, hi=6.0):
        n = len(self.g["nodes"])
        return self.node("Clip", [x, self.const("lo%d" % n, [lo]), self.const("hi%d" % n, [hi])])

    def done(self, *outs):
        self.g["outputs"] = [(o, []) for o in outs]
        return self.g


def graph_pads():
    """Pads: reflect, edge and constant, folded (symmetric, stride 2, asymmetric begin / end) and standalone (two consumers, asymmetric);
    Conv k = 1, 2, 3, 5 with and without bias, own symmetric and TF-style asymmetric pads; fused Relu, LeakyRelu, Tanh, Sigmoid; MaxPool,
    AveragePool, Concat."""
    b = Graph("pads", 4, 19, 23, 1)
    y = b.node("Relu", [b.conv(b.pad("x", 1, 1, 1, 1, "reflect"), 8, 3)])
    y = b.node("LeakyRelu", [b.conv(b.pad(y, 2, 2, 2, 2, "edge"), 8, 5, 2, bias=False)], {"alpha": 0.2})
    y = b.node("Tanh", [b.conv(b.pad(y, 0, 1, 0, 1), 8, 2)])
    y = b.node("Sigmoid", [b.conv(y, 8, 3, 2, pads=(0, 0, 1, 1))])  # ONNX pads [t, l, b, r]: TF's stride-2 'same'
    p = b.pad(y, 1, 0, 1, 2, "edge")  # two consumers: standalone
    m = b.node("MaxPool", [p], {"kernel_shape": [2, 2], "strides": [2, 2]})
    c = b.conv(p, 8, 3, pads=(1, 1, 1, 1), bias=False)
    a = b.node("AveragePool", [c], {"kernel_shape": [2, 2], "strides": [2, 2]})
    q = b.pad(b.node("Concat", [m, a], {"axis": 1}, planes=16), 2, 2, 2, 2, "reflect")  # standalone: its consumer is not a Conv
    return b.done(b.conv(b.node("AveragePool", [q], {"kernel_shape": [3, 3], "strides": [3, 3]}), 8, 1))


def graph_depthwise_bn():
    """Depthwise stride 1 (own pads) and 2 (a folded constant Pad) with folded BN and Clip (relu6), BN folded and standalone at eps 1e-5
    and 1e-3, standalone Clip / Sigmoid / Tanh, InstanceNorm on small activations, Add with a fused Relu."""
    b = Graph("depthwise_bn", 8, 21, 18, 2)
    y = b.clip(b.bn(b.conv("x", 16, 1), 1e-5))
    y = b.clip(b.bn(b.conv(y, 16, 3, 1, pads=(1, 1, 1, 1), bias=False, group=16), 1e-3))
    y = b.node("Relu", [b.conv(b.pad(y, 1, 1, 1, 1), 16, 3, 2, group=16)])
    c = b.conv(y, 16, 1)  # two consumers: the BNs below stay standalone
    s = b.node("Sigmoid", [b.bn(c, 1e-3)])
    t = b.node("Tanh", [b.bn(c, 1e-5)])
    z = b.node("Relu", [b.node("Add", [s, t])])
    n = b.instance_norm(b.conv(z, 8, 3, pads=(1, 1, 1, 1), gain=0.02))  # variances ~1e-4 .. 1e-3: the epsilon matters
    m = b.node("MaxPool", [b.pad(z, 1, 1, 1, 1)], {"kernel_shape": [2, 2], "strides": [2, 2]})  # a standalone constant Pad
    return b.done(b.clip(b.node("Add", [n, b.conv(z, 8, 1, bias=False)])), m)


def graph_resize():
    """Resize / Upsample: nearest x2 (Resize half_pixel, Resize asymmetric floor, Upsample), linear x2 (half_pixel, pytorch_half_pixel),
    linear x1.5 (half_pixel), linear x1 (every coordinate mode); standalone Relu, LeakyRelu, Tanh, Sigmoid and Clip."""
    b = Graph("resize", 6, 9, 11, 3)
    c = b.conv("x", 8, 3, pads=(1, 1, 1, 1))
    n1 = b.node("Relu", [b.resize(c, 2, "nearest")])
    n2 = b.resize(c, 2, "nearest", "asymmetric", "floor")
    n3 = b.resize(c, 2, "nearest", op="Upsample")
    l1 = b.node("LeakyRelu", [b.resize(c, 2, "linear", "half_pixel")], {"alpha": 0.1})
    l2 = b.resize(c, 2, "linear", "pytorch_half_pixel")
    up = b.node("Add", [b.node("Add", [n1, n2]), b.node("Add", [n3, b.node("Add", [l1, l2])])])
    f = b.clip(b.resize(c, 1.5, "linear", "half_pixel"))
    one = [b.resize(c, 1, "linear", m) for m in ("half_pixel", "asymmetric", "align_corners")]
    k = b.node("Tanh", [b.node("Add", [b.node("Add", one[:2]), one[2]])])
    return b.done(b.node("Sigmoid", [b.node("Concat", [b.conv(up, 8, 5, 2, pads=(2, 2, 2, 2)), b.conv(k, 8, 1)], {"axis": 1}, planes=16)]), f)


GRAPHS = {"pads": graph_pads, "depthwise_bn": graph_depthwise_bn, "resize": graph_resize}
GRAPH_INPUT = {"pads": (2, 19, 23, 4), "depthwise_bn": (2, 21, 18, 8), "resize": (2, 9, 11, 6)}


def graph_input(name, seed=0):
    return np.random.default_rng(seed).uniform(-1, 1, GRAPH_INPUT[name]).astype(np.float32)


def _one(op_fn):
    b = Graph("refused", 8, 16, 16, 7)
    return b.done(op_fn(b))


# graphs the converter must refuse, with the attribute the ValueError must name
REFUSED = {
    "depthwise asymmetric pads": (lambda: _one(lambda b: b.conv("x", 8, 3, 2, pads=(0, 0, 1, 1), group=8)), "pads"),
    "conv pads differ between the axes": (lambda: _one(lambda b: b.conv("x", 8, 3, 1, pads=(1, 0, 1, 2))), "pads"),
    "1x1 conv with pads": (lambda: _one(lambda b: b.conv("x", 8, 1, 1, pads=(1, 1, 1, 1))), "pads"),
    "unpadded 3x3 conv": (lambda: _one(lambda b: b.conv("x", 8, 3)), "pads"),
    "even kernel, stride 1, no pads": (lambda: _one(lambda b: b.conv("x", 8, 2)), "pads"),
    "Pad T != L": (lambda: _one(lambda b: b.node("Relu", [b.pad("x", 1, 1, 0, 0)])), "pads"),
    "Pad wrap": (lambda: _one(lambda b: b.node("Relu", [b.pad("x", 1, 1, 1, 1, "wrap")])), "mode"),
    "Pad constant value": (lambda: _one(lambda b: b.node("Relu", [b.node("Pad", ["x"], {"mode": "constant", "pads": [0, 0, 1, 1, 0, 0, 1, 1], "value": 1.0})])),
                           "value"),
    "MaxPool pads": (lambda: _one(lambda b: b.node("MaxPool", ["x"], {"kernel_shape": [3, 3], "strides": [2, 2], "pads": [1, 1, 1, 1]})), "pads"),
    "AveragePool pads": (lambda: _one(lambda b: b.node("AveragePool", ["x"], {"kernel_shape": [2, 2], "strides": [2, 2], "pads": [0, 0, 1, 1]})), "pads"),
    "MaxPool 3x3 stride 2": (lambda: _one(lambda b: b.node("MaxPool", ["x"], {"kernel_shape": [3, 3], "strides": [2, 2]})), "strides"),
    "Resize linear asymmetric": (lambda: _one(lambda b: b.resize("x", 2, "linear", "asymmetric")), "coordinate_transformation_mode"),
    "Resize linear align_corners": (lambda: _one(lambda b: b.resize("x", 2, "linear", "align_corners")), "coordinate_transformation_mode"),
    "Upsample linear": (lambda: _one(lambda b: b.resize("x", 2, "linear", op="Upsample")), "coordinate_transformation_mode"),
    "Resize nearest x1.5": (lambda: _one(lambda b: b.resize("x", 1.5, "nearest")), "scale"),
    "Resize nearest x3 asymmetric round": (lambda: _one(lambda b: b.resize("x", 3, "nearest", "asymmetric")), "nearest_mode"),
    "Resize nearest x2 align_corners": (lambda: _one(lambda b: b.resize("x", 2, "nearest", "align_corners", "floor")), "coordinate_transformation_mode"),
    "Resize cubic": (lambda: _one(lambda b: b.resize("x", 2, "cubic")), "mode"),
    "InstanceNormalization epsilon": (lambda: _one(lambda b: b.instance_norm("x", 1e-3)), "epsilon"),
    "Clip min / max": (lambda: _one(lambda b: b.clip(b.conv("x", 8, 3, pads=(1, 1, 1, 1)), -1.0, 1.0)), "min"),
}


def candy_input(n, h, w, seed=0):
    """Input at the real Candy model's 0..255 scale."""
    return np.random.default_rng(seed).uniform(0, 255, (n, h, w, 3)).astype(np.float32)


# the real Candy head's cases: (fold_pads, (h, w), batch)
CANDY = [(fold, hw, n) for fold in (True, False) for hw, n in (((64, 64), 1), ((70, 131), 2))]
