"""Writers of SNN JSON model files (the format core/src/ic2/modelparser.cpp reads; SURVEY.md Appendix B).

Every model JSON in the reference's modelzoo/ is a Git-LFS pointer stub (SURVEY F4), so the BASELINE configs are
rebuilt here from the architecture files that DO exist (ncnn .param graphs, demo/modelInferenceESPCN.py) with
deterministic synthetic weights. This is the writer side of the format, i.e. what tools/convertTool emits
(h5ToJsonConverter.py:101-114,168-190): either one JSON with embedded weight arrays, or `<model>_layers.json` +
`<model>_weights.bin` (raw LE fp32 in layer order: kernel, bias (if useBias), gamma, beta, mean, var (if BN)).

Layer dict conventions == the JSON keys; weights live under the private key "_w" until written.
"""
import json
import os

import numpy as np

SEED = 7767517  # the seed every reference op test uses (demo/test/unittest/convolutionTest.cpp:417)


class Builder:
    def __init__(self, seed=SEED):
        self.layers = []
        self.rng = np.random.default_rng(seed)

    # -- synthetic weight distributions (SURVEY §8d): He-normal kernels, small biases, BN near identity --
    def _kernel(self, oc, ic, k, gain=2.0, bn=False):
        # a BatchNorm with gamma in U[0.5,1.5] and variance in U[0.5,1.5] multiplies the output's second moment by
        # E[gamma^2] * E[1/var] = 1.083 * ln(3) = 1.19: taken out of the kernel so that activations stay O(1) through depth
        std = np.sqrt(gain / (1.19 if bn else 1.0) / (k * k * ic))
        return (self.rng.standard_normal((oc, ic, k, k)) * std).astype(np.float32)

    def _bias(self, c):
        return self.rng.uniform(-0.1, 0.1, c).astype(np.float32)

    def _bn(self, c):
        return {
            "gamma": self.rng.uniform(0.5, 1.5, c).astype(np.float32),
            "beta": self.rng.uniform(-0.1, 0.1, c).astype(np.float32),
            "moving_mean": self.rng.uniform(-0.1, 0.1, c).astype(np.float32),
            "moving_variance": self.rng.uniform(0.5, 1.5, c).astype(np.float32),
        }

    def _add(self, d, inputs):
        d["numInputs"] = len(inputs)
        d["inputId"] = list(inputs)
        self.layers.append(d)
        return len(self.layers) - 1

    def planes(self, i):
        return self.layers[i]["outputPlanes"]

    def input(self, w, h, c, index=0):
        return self._add({"type": "InputLayer", "name": "input_%d" % (index + 1), "Input Width": w, "Input Height": h, "outputPlanes": c,
                          "inputPlanes": c, "inputIndex": index}, [])

    def conv(self, x, oc, k, stride=1, padding="same", activation="linear", bias=True, bn=False, alpha=None, mode=None, gain=2.0):
        ic = self.planes(x)
        d = {"type": "Conv2D", "name": "conv2d_%d" % len(self.layers), "inputPlanes": ic, "outputPlanes": oc, "kernel_size": k, "strides": stride,
             "padding": padding, "activation": activation, "useBias": "True" if bias else "False",
             "useBatchNormalization": "True" if bn else "False"}
        if mode is not None:
            d["mode"] = mode
        if activation == "leakyRelu":
            d["leakyReluAlpha"] = 0.1 if alpha is None else alpha
        w = {"kernel": self._kernel(oc, ic, k, gain, bn)}
        if bias:
            w["bias"] = self._bias(oc)
        d["_w"] = w
        if bn:
            d["_bn"] = self._bn(oc)
        return self._add(d, [x])

    def depthwise(self, x, k=3, stride=1, padding="same", activation="linear", bias=False, bn=True):
        c = self.planes(x)
        d = {"type": "DepthwiseConv2D", "name": "depthwise_conv2d_%d" % len(self.layers), "inputPlanes": c, "outputPlanes": c, "kernel_size": k,
             "strides": stride, "padding": padding, "activation": activation, "useBias": "True" if bias else "False",
             "useBatchNormalization": "True" if bn else "False"}
        std = np.sqrt(2.0 / (1.19 if bn else 1.0) / (k * k))
        w = {"kernel_chw": (self.rng.standard_normal((c, k, k)) * std).astype(np.float32)}  # canonical [C][kh][kw]
        if bias:
            w["bias"] = self._bias(c)
        d["_w"] = w
        if bn:
            d["_bn"] = self._bn(c)
        return self._add(d, [x])

    def maxpool(self, x, k, stride=None, padding="valid"):
        c = self.planes(x)
        return self._add({"type": "MaxPooling2D", "name": "max_pooling2d_%d" % len(self.layers), "inputPlanes": c, "outputPlanes": c, "pool": [k, k],
                          "strides": stride if stride is not None else k, "padding": padding}, [x])

    def avgpool(self, x, k, stride=None, padding="valid"):
        c = self.planes(x)
        return self._add({"type": "AveragePooling2D", "name": "average_pooling2d_%d" % len(self.layers), "inputPlanes": c, "outputPlanes": c,
                          "pool_size": [k, k], "stride": stride if stride is not None else k, "padding": padding}, [x])

    def global_avgpool(self, x, size):
        """What the converter emits for a global pool (averagepooling2d.py:40-55): pool_size=[H,H], strides=[1,1], valid.
        The reader ignores "strides" for average pools, so the stride defaults to the pool size -> 1x1 output."""
        c = self.planes(x)
        return self._add({"type": "AveragePooling2D", "name": "global_average_pooling2d_%d" % len(self.layers), "inputPlanes": c, "outputPlanes": c,
                          "pool_size": [size, size], "strides": [1, 1], "padding": "valid"}, [x])

    def add(self, a, b, activation="linear"):
        c = self.planes(a)
        return self._add({"type": "Add", "name": "add_%d" % len(self.layers), "inputPlanes": c, "outputPlanes": c, "activation": activation}, [a, b])

    def flatten(self, x, planes):
        return self._add({"type": "Flatten", "name": "flatten", "inputPlanes": self.planes(x), "outputPlanes": planes}, [x])

    def dense(self, x, n_in, units, activation="softmax", bias=True):
        std = np.sqrt(1.0 / n_in)
        w = {"kernel": (self.rng.standard_normal((units, n_in)) * std).astype(np.float32)}  # [out][in] (cpulayer.h:162)
        if bias:
            w["bias"] = self._bias(units)
        return self._add({"type": "Dense", "name": "dense", "inputPlanes": n_in, "outputPlanes": units, "units": units, "activation": activation,
                          "useBias": "True" if bias else "False", "_w": w}, [x])

    def pad(self, x, t, b, l, r, mode=None):
        c = self.planes(x)
        d = {"type": "ZeroPadding2D", "name": "zero_padding2d_%d" % len(self.layers), "inputPlanes": c, "outputPlanes": c, "padding": [[t, b], [l, r]]}
        if mode:
            d["mode"] = mode
        return self._add(d, [x])

    def upsample(self, x, scale=2, interpolation="nearest"):
        c = self.planes(x)
        return self._add({"type": "UpSampling2D", "name": "up_sampling2d_%d" % len(self.layers), "inputPlanes": c, "outputPlanes": c, "scaleFactor": scale,
                          "interpolation": interpolation}, [x])

    def concat(self, a, b):
        c = self.planes(a) + self.planes(b)
        return self._add({"type": "Concatenate", "name": "concatenate_%d" % len(self.layers), "inputPlanes": self.planes(a), "outputPlanes": c}, [a, b])

    def instancenorm(self, x, activation="linear"):
        c = self.planes(x)
        w = {"scale": self.rng.uniform(0.5, 1.5, c).astype(np.float32), "bias": self.rng.uniform(-0.1, 0.1, c).astype(np.float32)}
        return self._add({"type": "InstanceNormalization", "name": "instance_norm_%d" % len(self.layers), "inputPlanes": c, "outputPlanes": c,
                          "epsilon": 1e-5, "activation": activation, "_w": w}, [x])

    def batchnorm(self, x, activation="linear"):
        c = self.planes(x)
        return self._add({"type": "BatchNormalization", "name": "batch_normalization_%d" % len(self.layers), "inputPlanes": c, "outputPlanes": c,
                          "activation": activation, "_bn": self._bn(c)}, [x])

    def subpixel(self, x, r=2):
        return self._add({"type": "Lambda", "name": "subpixel", "inputPlanes": self.planes(x), "outputPlanes": 1, "kernel_size": r}, [x])

    def yolo(self, a, b):
        return self._add({"type": "YOLO", "name": "yolo", "inputPlanes": self.planes(a), "outputPlanes": 6}, [a, b])


# ----------------------------------------------------------------------------------------------------------------
# writers
# ----------------------------------------------------------------------------------------------------------------
def _tolist(a):
    return [float(v) for v in np.asarray(a, dtype=np.float32).ravel()]


def write_model(layers, path, split=False):
    """Write `layers` to `path` (JSON). split=True streams the weights to `<stem>_weights.bin` next to it
    (tools/convertTool onnxToJsonConverter.py:69-73 naming) and names it in numLayers.bin_file_name."""
    os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
    root = {"numLayers": {"count": len(layers)}}
    binf = None
    if split:
        stem = os.path.basename(path)
        stem = stem[:-len("_layers.json")] if stem.endswith("_layers.json") else os.path.splitext(stem)[0]
        bin_name = stem + "_weights.bin"
        root["numLayers"]["bin_file_name"] = bin_name
        binf = open(os.path.join(os.path.dirname(os.path.abspath(path)), bin_name), "wb")

    def put(arr):
        binf.write(np.ascontiguousarray(arr, dtype="<f4").tobytes())

    for i, l in enumerate(layers):
        d = {k: v for k, v in l.items() if not k.startswith("_")}
        w = l.get("_w")
        bn = l.get("_bn")
        t = l["type"]
        if t == "Conv2D":
            if split:
                put(w["kernel"])  # OIHW (modelparser.cpp:621-637)
                if "bias" in w:
                    put(w["bias"])
                d["weights"] = {}
            else:
                d["weights"] = {"kernel": _tolist(w["kernel"])}
                if "bias" in w:
                    d["weights"]["bias"] = _tolist(w["bias"])
        elif t in ("DepthwiseConv2D", "Depthwise", "SeparableConv2D"):
            chw = w["kernel_chw"]
            if split:
                put(chw)  # .bin variant is [C][kh][kw] (modelparser.cpp:827-840)
                if "bias" in w:
                    put(w["bias"])
                d["weights"] = {}
            else:
                c, k, _ = chw.shape
                d["weights"] = {"kernel": _tolist(chw.reshape(c, k * k).T)}  # JSON flat = [kh*kw][C] (modelparser.cpp:843-850)
                if "bias" in w:
                    d["weights"]["bias"] = _tolist(w["bias"])
        elif t == "Dense":
            if split:
                put(w["kernel"])
                if "bias" in w:
                    put(w["bias"])
                d["weights"] = {}
            else:
                d["weights"] = {"kernel": _tolist(w["kernel"])}
                if "bias" in w:
                    d["weights"]["bias"] = _tolist(w["bias"])
        elif t in ("InstanceNormalization", "InstanceNorm"):
            d["weights"] = {"scale": _tolist(w["scale"]), "bias": _tolist(w["bias"])}  # always embedded (modelparser.cpp:1166-1185)
        if bn is not None:
            if split and t != "BatchNormalization":
                for key in ("gamma", "beta", "moving_mean", "moving_variance"):  # modelparser.cpp:694-726
                    put(bn[key])
                d["batchNormalization"] = {}
            else:
                d["batchNormalization"] = {k: _tolist(v) for k, v in bn.items()}
        root["Layer_%d" % i] = d
    if binf:
        binf.close()
    with open(path, "w") as f:
        json.dump(root, f)
    return path


# ----------------------------------------------------------------------------------------------------------------
# torch-CPU evaluation of a layer list (writer-side tool, NOT a product path: the engine never imports it).
# Used (a) to calibrate the classifier heads of the synthetic models on data (LSUV-style: logits centred and O(1), so the
# arg-max differs from image to image and the softmax is not saturated) and (b) by tests/ as a third, independent
# implementation of the BASELINE graphs at full size next to the oracle and the CUDA engine. Covers the layer types of
# the two classification graphs and of Candy / YOLO bodies; anything else raises.
# ----------------------------------------------------------------------------------------------------------------
def _pad4(l, k):
    """[T, B, L, R] of a conv/pad layer dict (conv2d.cpp:39-74 semantics)."""
    p = l.get("padding", "valid")
    if isinstance(p, list):
        if isinstance(p[0], list):
            return [int(p[0][0]), int(p[0][1]), int(p[1][0]), int(p[1][1])]
        return [int(p[0]), int(p[0]), int(p[1]), int(p[1])]
    if isinstance(p, (int, float)):
        return [int(p)] * 4
    if p in ("valid", "none") or k <= 1:
        return [0, 0, 0, 0]
    o = [k // 2] * 4
    if k % 2 == 0:
        o[0] -= 1
        o[2] -= 1
    return o


def torch_forward(layers, x_nhwc, upto=None):
    """Evaluate `layers` (Builder dicts with "_w"/"_bn") on an NHWC fp32 batch with torch-CPU ops in fp64-free fp32.
    Returns the list of NHWC numpy outputs (None past `upto`)."""
    import torch
    import torch.nn.functional as F

    def act(y, l):
        a = l.get("activation", "linear")
        if a == "relu":
            return F.relu(y)
        if a == "relu6":
            return torch.clamp(y, 0.0, 6.0)
        if a == "tanh":
            return torch.tanh(y)
        if a == "sigmoid":
            return torch.sigmoid(y)
        if a in ("leakyRelu", "leaky_relu"):
            return torch.maximum(y, y * float(l.get("leakyReluAlpha", l.get("alpha", 0.3))))
        if a == "softmax":
            return torch.softmax(y, dim=1)
        return y

    def bn(y, d):
        if d is None:
            return y
        t = lambda k: torch.from_numpy(np.asarray(d[k], np.float32)).view(1, -1, 1, 1)
        s = torch.clamp(torch.sqrt(t("moving_variance") + 1e-3), min=1e-4)
        return t("gamma") / s * (y - t("moving_mean")) + t("beta")

    outs = [None] * len(layers)
    with torch.no_grad():
        for i, l in enumerate(layers):
            if upto is not None and i > upto:
                break
            t = l["type"]
            ins = [outs[j] for j in l.get("inputId", [])]
            w = l.get("_w", {})
            if t == "InputLayer":
                y = torch.from_numpy(np.ascontiguousarray(x_nhwc, dtype=np.float32)).permute(0, 3, 1, 2).contiguous()
            elif t == "Conv2D":
                k, s = int(l["kernel_size"]), int(l["strides"])
                o = _pad4(l, k)
                mode = l.get("mode", "constant") if any(o) else "constant"
                a = F.pad(ins[0], (o[2], o[3], o[0], o[1]), mode={"constant": "constant", "reflect": "reflect", "replicate": "replicate"}[mode])
                y = F.conv2d(a, torch.from_numpy(w["kernel"]), torch.from_numpy(w["bias"]) if "bias" in w else None, stride=s)
                y = act(bn(y, l.get("_bn")), l)
            elif t in ("DepthwiseConv2D", "Depthwise", "SeparableConv2D"):
                k, s = int(l["kernel_size"]), int(l["strides"])
                o = _pad4(l, k)
                a = F.pad(ins[0], (o[2], o[3], o[0], o[1]))
                c = a.shape[1]
                y = F.conv2d(a, torch.from_numpy(w["kernel_chw"]).view(c, 1, k, k), torch.from_numpy(w["bias"]) if "bias" in w else None, stride=s, groups=c)
                y = act(bn(y, l.get("_bn")), l)
            elif t in ("MaxPooling2D", "AveragePooling2D"):
                pool = l.get("pool", l.get("pool_size"))
                k = int(pool[0] if isinstance(pool, list) else pool)
                s = l.get("stride", l.get("strides", k)) if t == "MaxPooling2D" else l.get("stride", k)
                s = int(s[0] if isinstance(s, list) else s)
                a = ins[0]
                h, wd = a.shape[2], a.shape[3]
                valid = str(l.get("padding")) in ("0", "valid", "none")
                od = lambda n: int(np.float32(n) / np.float32(s) + 1.0 - (np.float32(k) / np.float32(s) if valid else 1.0 / np.float32(s)))
                oh, ow = od(h), od(wd)
                # windows start at o*s and are clipped at the bottom/right edge, never padded top/left (maxpool2dVulkan.cpp:54-60)
                pb, pr = max(0, (oh - 1) * s + k - h), max(0, (ow - 1) * s + k - wd)
                if t == "MaxPooling2D":
                    y = F.max_pool2d(F.pad(a, (0, pr, 0, pb), value=float("-inf")), k, s)[:, :, :oh, :ow]
                else:
                    ones = F.pad(torch.ones_like(a[:, :1]), (0, pr, 0, pb))
                    y = (F.avg_pool2d(F.pad(a, (0, pr, 0, pb)), k, s) / F.avg_pool2d(ones, k, s))[:, :, :oh, :ow]
            elif t == "Add":
                y = act(ins[0] + ins[1], l)
            elif t in ("ZeroPadding2D", "Pad"):
                o = _pad4(l, 0)
                y = F.pad(ins[0], (o[2], o[3], o[0], o[1]), mode={"constant": "constant", "reflect": "reflect", "replicate": "replicate"}[l.get("mode", "constant")])
            elif t == "Flatten":
                y = ins[0].permute(0, 2, 3, 1).reshape(ins[0].shape[0], -1, 1, 1)  # HWC order (cpulayer.h:94-115)
            elif t == "Dense":
                a = ins[0].permute(0, 2, 3, 1).reshape(ins[0].shape[0], -1)
                y = a @ torch.from_numpy(w["kernel"]).t()
                if "bias" in w:
                    y = y + torch.from_numpy(w["bias"])
                y = act(y, l).view(a.shape[0], -1, 1, 1)
            elif t in ("InstanceNormalization", "InstanceNorm"):
                a = ins[0]
                m, v = a.mean(dim=(2, 3), keepdim=True), a.var(dim=(2, 3), unbiased=False, keepdim=True)
                y = (a - m) / torch.sqrt(v + 1e-5) * torch.from_numpy(w["scale"]).view(1, -1, 1, 1) + torch.from_numpy(w["bias"]).view(1, -1, 1, 1)
                y = act(y, l)
            elif t == "UpSampling2D" and l.get("interpolation", "nearest") == "nearest":
                y = F.interpolate(ins[0], scale_factor=int(l["scaleFactor"]), mode="nearest")
            elif t == "Concatenate":
                y = torch.cat([ins[0], ins[1]], dim=1)
            elif t == "BatchNormalization":
                y = act(bn(ins[0], l.get("_bn")), l)
            else:
                raise NotImplementedError("torch_forward: layer type %s" % t)
            outs[i] = y
    return [None if o is None else o.permute(0, 2, 3, 1).contiguous().numpy() for o in outs]


def calibrate_head(layers, name, input_hw, images=8, logit_std=2.0):
    """Data-dependent init of the final Dense (the LSUV idea): on `images` calibration images (their own seed) compute the
    features g entering the Dense, then scale the kernel so that the image-dependent part of the logits has standard
    deviation `logit_std` and set the bias to -W.mean(g): logits are centred, the soft-max is far from saturation and the
    arg-max is decided by the image, not by a constant offset. Needs torch (CPU); a no-op without it."""
    try:
        import torch  # noqa: F401
    except Exception:
        return False
    di = max(i for i, l in enumerate(layers) if l["type"] == "Dense")
    x = synthetic_input(name, images, input_hw, seed=SEED + 1000)
    g = torch_forward(layers, x, upto=layers[di]["inputId"][0])[layers[di]["inputId"][0]].reshape(images, -1).astype(np.float64)
    w = layers[di]["_w"]["kernel"].astype(np.float64)
    gm = g.mean(0)
    var = ((g - gm) @ w.T).std()
    w *= logit_std / max(var, 1e-12)
    layers[di]["_w"]["kernel"] = w.astype(np.float32)
    layers[di]["_w"]["bias"] = (-(w @ gm)).astype(np.float32)
    layers[di]["useBias"] = "True"
    return True


# ----------------------------------------------------------------------------------------------------------------
# the BASELINE.json configurations
# ----------------------------------------------------------------------------------------------------------------
def resnet18(input_hw=(224, 224), classes=10, seed=SEED, calibrate=True, head_activation="softmax"):
    """modelzoo/Resnet18/resnet18_cifar10_0223.param (SURVEY App. D): Keras CIFAR variant — bias on every conv, the
    first block's first conv has no BN/ReLU, 1x1-s2 shortcuts with bias and no BN, Add then ReLU; at 224x224 the
    trailing AveragePooling2D(1,1) becomes the 7x7 global pool so Dense(512->classes) type-checks (SURVEY F6)."""
    b = Builder(seed)
    h, w = input_hw
    x = b.input(w, h, 3)
    x = b.conv(x, 64, 7, 2, "same", "relu", bias=True, bn=True)
    x = b.maxpool(x, 3, 2, "same")
    # Residual gains (SURVEY 8d: activations must stay O(1) so that relative error and the arg-max mean something): the
    # branch's last conv has gain 0.25 and a down-sampling shortcut gain 1, so that E[(x + y)^2] stays near E[x^2].
    # stage 1
    y = b.conv(x, 64, 3, 1, "same", "linear", bias=True, bn=False, gain=1.0)
    y = b.conv(y, 64, 3, 1, "same", "linear", bias=True, bn=True, gain=0.25)
    x = b.add(y, x, "relu")
    y = b.conv(x, 64, 3, 1, "same", "relu", bias=True, bn=True)
    y = b.conv(y, 64, 3, 1, "same", "linear", bias=True, bn=True, gain=0.25)
    x = b.add(y, x, "relu")
    for oc in (128, 256, 512):
        y = b.conv(x, oc, 3, 2, "same", "relu", bias=True, bn=True)
        y = b.conv(y, oc, 3, 1, "same", "linear", bias=True, bn=True, gain=0.5)
        s = b.conv(x, oc, 1, 2, "valid", "linear", bias=True, bn=False, gain=1.0)
        x = b.add(s, y, "relu")
        y = b.conv(x, oc, 3, 1, "same", "relu", bias=True, bn=True)
        y = b.conv(y, oc, 3, 1, "same", "linear", bias=True, bn=True, gain=0.25)
        x = b.add(y, x, "relu")
    x = b.global_avgpool(x, max(1, h // 32))
    x = b.flatten(x, 512)
    x = b.dense(x, 512, classes, head_activation)
    if calibrate:
        calibrate_head(b.layers, "resnet18", input_hw)
    return b.layers


def mobilenetv2(input_hw=(224, 224), classes=1000, seed=SEED, calibrate=True, head_activation="softmax"):
    """modelzoo/MobileNetV2/mobilenetV2.param (Keras, alpha=1): 3x3-s2 stem, 17 inverted-residual blocks (1x1 expand +BN
    +ReLU6 -> dw3x3 +BN +ReLU6 -> 1x1 project +BN), stride-2 depthwise behind ZeroPadding2D((0,1),(0,1)) + valid, 10
    residual adds, 1x1 320->1280 +BN +ReLU6, global average pool, classifier."""
    b = Builder(seed)
    h, w = input_hw
    x = b.input(w, h, 3)
    x = b.pad(x, 0, 1, 0, 1)
    x = b.conv(x, 32, 3, 2, "valid", "relu6", bias=False, bn=True)
    cfg = [(1, 16, 1, 1), (6, 24, 2, 2), (6, 32, 3, 2), (6, 64, 4, 2), (6, 96, 3, 1), (6, 160, 3, 2), (6, 320, 1, 1)]
    cin = 32
    first = True
    for t, c, n, s in cfg:
        for i in range(n):
            stride = s if i == 0 else 1
            inp = x
            # the reference graph keeps a 1x1 32->32 "expand" in the very first block (mobilenetV2.param conv2d_1)
            y = b.conv(x, cin * t if not first else cin, 1, 1, "valid", "relu6", bias=False, bn=True)
            first = False
            if stride == 2:
                y = b.pad(y, 0, 1, 0, 1)
                y = b.depthwise(y, 3, 2, "valid", "relu6", bias=False, bn=True)
            else:
                y = b.depthwise(y, 3, 1, "same", "relu6", bias=False, bn=True)
            y = b.conv(y, c, 1, 1, "valid", "linear", bias=False, bn=True, gain=1.0)
            x = b.add(y, inp, "linear") if (stride == 1 and cin == c) else y
            cin = c
    x = b.conv(x, 1280, 1, 1, "valid", "relu6", bias=False, bn=True)
    x = b.global_avgpool(x, max(1, h // 32))
    x = b.flatten(x, 1280)
    x = b.dense(x, 1280, classes, head_activation)
    if calibrate:
        calibrate_head(b.layers, "mobilenetv2", input_hw)
    return b.layers


def yolov3_tiny(input_hw=(416, 416), head_channels=18, seed=SEED):
    """modelzoo/Yolov3-tiny/yolov3-tiny_finetuned.param: 3x3 conv +BN +LeakyReLU(0.1) x7 with 2x2-s2 max pools (the last
    pool is 2x2 stride 1 'same'), 1x1 heads (bias, linear), nearest x2 upsample, concat(128 + 256), YOLO decode over the
    two heads. head_channels = 3*(5+classes): 18 for the 1-class decode the reference hard-codes (yololayer.cpp:31-38),
    255 for the COCO heads of the .param file."""
    b = Builder(seed)
    h, w = input_hw
    x = b.input(w, h, 3)

    def cbl(x, oc, k):
        return b.conv(x, oc, k, 1, "same" if k > 1 else "valid", "leakyRelu", bias=False, bn=True, alpha=0.1)

    x = cbl(x, 16, 3)
    x = b.maxpool(x, 2, 2, "valid")
    x = cbl(x, 32, 3)
    x = b.maxpool(x, 2, 2, "valid")
    x = cbl(x, 64, 3)
    x = b.maxpool(x, 2, 2, "valid")
    x = cbl(x, 128, 3)
    x = b.maxpool(x, 2, 2, "valid")
    route_a = cbl(x, 256, 3)
    x = b.maxpool(route_a, 2, 2, "valid")
    x = cbl(x, 512, 3)
    x = b.maxpool(x, 2, 1, "same")
    x = cbl(x, 1024, 3)
    route_b = cbl(x, 256, 1)
    y = cbl(route_b, 512, 3)
    def head(t):
        # objectness biased low, as in a trained detector (a handful of cells pass the 0.35 confidence threshold, not thousands:
        # with random heads the host NMS, quadratic in the candidate count, was all the end-to-end number measured)
        i = b.conv(t, head_channels, 1, 1, "valid", "linear", bias=True, bn=False, gain=1.0)
        b.layers[i]["_w"]["bias"][4::head_channels // 3] = -2.0
        return i

    head13 = head(y)
    z = cbl(route_b, 128, 1)
    z = b.upsample(z, 2, "nearest")
    z = b.concat(z, route_a)
    z = cbl(z, 256, 3)
    head26 = head(z)
    b.yolo(head13, head26)
    return b.layers


def candy(input_hw=(720, 720), seed=SEED):
    """modelzoo/StyleTransfer/candy-9_simplified-opt.param topology (fast-neural-style): reflect-pad + conv9x9(3->32) ->
    IN+ReLU -> [reflect-pad + conv3x3 s2] x2 (64, 128) -> 5 residual blocks (pad+conv3x3, IN, ReLU, pad+conv3x3, IN, add)
    -> [nearest x2, pad, conv3x3, IN, ReLU] x2 (64, 32) -> pad + conv9x9(32->3). Synthetic weights (the real ONNX weights
    are a next-round item, SURVEY §8f N1)."""
    b = Builder(seed)
    h, w = input_hw
    x = b.input(w, h, 3)

    def pconv(x, oc, k, stride):
        # the converter folds ReflectionPad into the conv: padding [[p,p],[p,p]] + "mode" (modelparser.cpp:584-594). A separate
        # Pad + "valid" conv would NOT shrink under the reference's dims rule (negative translation clamped at 0).
        p = k // 2
        return b.conv(x, oc, k, stride, [[p, p], [p, p]], "linear", bias=True, bn=False, mode="reflect", gain=1.0)

    x = b.instancenorm(pconv(x, 32, 9, 1), "relu")
    x = b.instancenorm(pconv(x, 64, 3, 2), "relu")
    x = b.instancenorm(pconv(x, 128, 3, 2), "relu")
    for _ in range(5):
        y = b.instancenorm(pconv(x, 128, 3, 1), "relu")
        y = b.instancenorm(pconv(y, 128, 3, 1), "linear")
        x = b.add(y, x, "linear")
    x = b.upsample(x, 2, "nearest")
    x = b.instancenorm(pconv(x, 64, 3, 1), "relu")
    x = b.upsample(x, 2, "nearest")
    x = b.instancenorm(pconv(x, 32, 3, 1), "relu")
    x = pconv(x, 3, 9, 1)
    return b.layers


def espcn(input_hw=(224, 224), seed=SEED):
    """demo/modelInferenceESPCN.py:49-71: conv5x5(1->16, relu) -> conv3x3(16->16, relu) -> conv3x3(16->4) ->
    depth_to_space(2) -> tanh (the Subpixel layer applies tanh itself, vk_subpixel.comp:64-66)."""
    b = Builder(seed)
    h, w = input_hw
    x = b.input(w, h, 1)
    x = b.conv(x, 16, 5, 1, "same", "relu", bias=True)
    x = b.conv(x, 16, 3, 1, "same", "relu", bias=True)
    x = b.conv(x, 4, 3, 1, "same", "linear", bias=True)
    x = b.subpixel(x, 2)
    return b.layers


def calibrate_segmentation_head(layers, input_hw, images=4, logit_std=2.0):
    """calibrate_head for the last (1x1) convolution of a segmentation model, on `images` calibration images (their own seed), with
    every pixel a sample: the kernel is scaled so that the logits' spread over pixels and images is `logit_std`, and the bias centres
    them. One output channel: the median pre-sigmoid value becomes 0, so the 0.5 threshold splits the pixels. Several: each class's
    logit is centred on its mean, so the arg-max is decided by the pixel's features. Needs torch (CPU); a no-op without it."""
    try:
        import torch  # noqa: F401
    except Exception:
        return False
    ci = max(i for i, l in enumerate(layers) if l["type"] == "Conv2D")
    src = layers[ci]["inputId"][0]
    x = synthetic_input("unet", images, input_hw, seed=SEED + 1000)
    g = torch_forward(layers, x, upto=src)[src].reshape(-1, layers[ci]["inputPlanes"]).astype(np.float64)
    w = layers[ci]["_w"]["kernel"][:, :, 0, 0].astype(np.float64)  # [K, C]
    z = (g - g.mean(0)) @ w.T
    w *= logit_std / max(float(z.std()), 1e-12)
    z = g @ w.T
    b = -np.median(z, axis=0) if w.shape[0] == 1 else -z.mean(0)
    layers[ci]["_w"]["kernel"] = w.astype(np.float32).reshape(layers[ci]["_w"]["kernel"].shape)
    layers[ci]["_w"]["bias"] = b.astype(np.float32)
    return True


def unet(input_hw=(256, 256), classes=1, seed=SEED, calibrate=True):
    """modelzoo/U-Net/unet.param (the grey-input U-Net of demo/test_unet.sh): [3x3 conv + ReLU] x2 at 64, 128, 256 and 512 channels,
    each followed by a 2x2 max pool, then [3x3 conv + ReLU] x2 at 1024; four decoder stages of nearest x2, a 2x2 'same' conv + ReLU at
    half the channels, concat(that, the encoder's output of that size) and [3x3 conv + ReLU] x2; head 3x3 conv 64->2 + ReLU, 1x1 conv
    2->1 + sigmoid. Every convolution has a bias and no BN. classes = K > 1 replaces the last two convolutions with one linear 1x1 conv
    64->K (a multi-class variant, not a reference graph). The last convolution is calibrated (calibrate_segmentation_head)."""
    b = Builder(seed)
    h, w = input_hw
    x = b.input(w, h, 1)

    def double(x, oc):
        x = b.conv(x, oc, 3, 1, "same", "relu", bias=True)
        return b.conv(x, oc, 3, 1, "same", "relu", bias=True)

    skips = []
    for oc in (64, 128, 256, 512):
        x = double(x, oc)
        skips.append(x)
        x = b.maxpool(x, 2, 2, "valid")
    x = double(x, 1024)
    for oc, skip in zip((512, 256, 128, 64), reversed(skips)):
        x = b.upsample(x, 2, "nearest")
        x = b.conv(x, oc, 2, 1, "same", "relu", bias=True)
        x = b.concat(x, skip)
        x = double(x, oc)
    if classes == 1:
        x = b.conv(x, 2, 3, 1, "same", "relu", bias=True)
        b.conv(x, 1, 1, 1, "valid", "sigmoid", bias=True, gain=1.0)
    else:
        b.conv(x, classes, 1, 1, "valid", "linear", bias=True, gain=1.0)
    if calibrate:
        calibrate_segmentation_head(b.layers, input_hw)
    return b.layers


MODELS = {
    "espcn": (espcn, (224, 224), 1, (0.0, 1.0)),
    "unet": (unet, (256, 256), 1, (0.0, 1.0)),
    "resnet18": (resnet18, (224, 224), 3, (-1.0, 1.0)),
    "mobilenetv2": (mobilenetv2, (224, 224), 3, (0.0, 1.0)),
    "yolov3tiny": (yolov3_tiny, (416, 416), 3, (-1.0, 1.0)),
    "candy": (candy, (720, 720), 3, (0.0, 255.0)),
}


def build(name, out_dir, input_hw=None, split=None, **kw):
    """Generate model `name` under out_dir; returns (json_path, layers). Large models default to the split
    (.json + _weights.bin) variant; ESPCN embeds its weights so both reader paths are exercised."""
    fn, hw, _, _ = MODELS[name]
    hw = tuple(input_hw) if input_hw else hw
    layers = fn(hw, **kw)
    if split is None:
        split = name != "espcn"
    fname = "%s_%dx%d%s.json" % (name, hw[0], hw[1], "_layers" if split else "")
    path = os.path.join(out_dir, fname)
    write_model(layers, path, split=split)
    return path, layers


def synthetic_input(name, batch, input_hw=None, seed=SEED):
    """Images in the model's normalised range (SURVEY 8d; constants of demo/common/modelInference.cpp). Every image has its
    own base colour, contrast and a few oriented gratings under the noise: i.i.d. noise images are statistically identical,
    which made every image of a batch land on the same class (VERDICT r1, weak #1)."""
    _, hw, c, (lo, hi) = MODELS[name]
    hw = tuple(input_hw) if input_hw else hw
    rng = np.random.default_rng(seed + 1)
    h, w = hw
    yy, xx = np.meshgrid(np.arange(h, dtype=np.float32) / h, np.arange(w, dtype=np.float32) / w, indexing="ij")
    out = np.empty((batch, h, w, c), np.float32)
    for n in range(batch):
        base = rng.uniform(0.15, 0.85, c).astype(np.float32)
        img = np.broadcast_to(base, (h, w, c)).copy()
        for _ in range(3):
            fx, fy = rng.uniform(-6.0, 6.0, 2)
            amp = rng.uniform(-0.25, 0.25, c).astype(np.float32)
            img += np.sin(2.0 * np.pi * (fx * xx + fy * yy) + rng.uniform(0, 6.28))[..., None].astype(np.float32) * amp
        img += rng.uniform(-1.0, 1.0, (h, w, c)).astype(np.float32) * np.float32(rng.uniform(0.02, 0.3))
        out[n] = np.clip(img, 0.0, 1.0)
    return (lo + (hi - lo) * out).astype(np.float32)
