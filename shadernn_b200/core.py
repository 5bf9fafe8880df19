"""Python mirror of the reference's public engine API over the C-ABI (numpy in, numpy out).

  GpuContext            ~ snn::GpuContext + dp::DeviceBackend            (core/inc/snn/snn.h, core/src/ic2/backend.h)
  ImageTexture          ~ snn::ImageTexture                              (core/inc/snn/imageTexture.h)
  MixedInferenceCore    ~ snn::MixedInferenceCore::create / run          (core/inc/snn/core.h:66-146)
  ShaderUnitTest-style single-layer helpers (conv2d, depthwise, ...)     (demo/common/shaderUnitTest.cpp:174-280)

Every call goes through libsnn_b200.so; nothing here computes.
"""
import ctypes as C
import sys
import weakref

import numpy as np

from . import _lib
from ._lib import ConvDesc, ModelOptions, check, lib, vp

ACT = {"": 0, "linear": 0, "identity": 0, "none": 0, "relu": 1, "relu6": 2, "tanh": 3, "sigmoid": 4, "leakyRelu": 5, "leaky_relu": 5, "SiLU": 6,
       "softmax": 7}
PAD_MODE = {"": 0, "none": 0, "constant": 1, "replicate": 2, "reflect": 3}
ALGO = {"auto": 0, "simt": 1, "tcgen05": 2, "tcgen05-streamk": 3}
PRECISION = {"fp32x3": 0, "fp16w": 1, "fp16": 2}


def _f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def _ptr(a):
    return None if a is None else a.ctypes.data_as(vp)


class GpuContext:
    def __init__(self, device=0):
        self.h = vp()
        check(lib().snnb_context_create(int(device), C.byref(self.h)), "snnb_context_create")
        self.device = device
        self._models = weakref.WeakSet()  # the open MixedInferenceCores on this context: destroying one uses its context

    def sync(self):
        check(lib().snnb_sync(self.h), "snnb_sync")

    def set_precision(self, precision):
        """Default product form of per-operator convolution launches: "fp32x3" (three bf16 MMAs) or "fp16w" (fp16 weights, two)."""
        check(lib().snnb_context_set_precision(self.h, PRECISION[precision]), "snnb_context_set_precision")

    def last_conv_variant(self):
        """snnb_debug_last_conv_variant: the instantiation of the most recent convolution launch on this context, as a dict with
        path ("simt", "igemm", "rowwin", "rowwin-feed"), terms, n_blk, ksplit, stream_k and fks."""
        out = (C.c_int * 6)()
        check(lib().snnb_debug_last_conv_variant(self.h, out), "snnb_debug_last_conv_variant")
        v = list(out)
        return {"path": ["none", "simt", "igemm", "rowwin", "rowwin-feed"][v[0]], "terms": v[1], "n_blk": v[2], "ksplit": v[3], "stream_k": v[4], "fks": v[5]}

    @property
    def stream(self):
        return lib().snnb_context_stream(self.h)

    @property
    def launches(self):
        return int(lib().snnb_launch_count(self.h))

    def rois_from_detections(self, rows, counts, frame_hw, capacity, min_score=0.0, class_id=-1, expand=0.0):
        """snnb_rois_from_detections: detect_frames / detect_torch rows (float32 CUDA [N, max_rows, 6]) and counts (int32 CUDA [N]) ->
        regions of frame_hw = (H, W) frames for MixedInferenceCore.run_rois, on the device, ordered on the current torch stream and
        never synchronising. Rows with score >= min_score and of class class_id (-1: any) are kept, each box grown by `expand` times its
        width (height) on each side and clipped to the frame, in frame order then row order. Returns (rois, count): an int32 CUDA tensor
        [capacity, 6] of {frame, row, x, y, width, height}, zero past the count, and an int32 CUDA tensor [1] with min(kept, capacity)."""
        import torch
        if not (isinstance(rows, torch.Tensor) and rows.is_cuda and rows.dtype == torch.float32 and rows.dim() == 3 and rows.shape[2] == 6):
            raise ValueError("rois_from_detections: rows must be a float32 CUDA tensor [N, max_rows, 6]")
        if not (isinstance(counts, torch.Tensor) and counts.is_cuda and counts.dtype == torch.int32 and tuple(counts.shape) == (rows.shape[0],)):
            raise ValueError("rois_from_detections: counts must be an int32 CUDA tensor [N] for rows of %d frames" % rows.shape[0])
        device = torch.device("cuda", self.device)
        rows, counts = rows.contiguous(), counts.contiguous()
        rois = torch.empty((max(int(capacity), 0), 6), dtype=torch.int32, device=device)
        count = torch.empty(1, dtype=torch.int32, device=device)
        sel = _lib.RoiSelect(float(min_score), int(class_id), float(expand))
        stream = torch.cuda.current_stream(device).cuda_stream or 1  # the legacy default stream is cudaStreamLegacy (1), not NULL
        check(lib().snnb_rois_from_detections(self.h, rows.data_ptr() or None, counts.data_ptr() or None, rows.shape[0], rows.shape[1], int(frame_hw[1]),
                                              int(frame_hw[0]), C.byref(sel), rois.data_ptr() or None, int(capacity), count.data_ptr(), stream),
              "snnb_rois_from_detections")
        return rois, count

    def close(self):
        """Destroys the context, after closing every model still open on it (snnb_model_destroy needs the context; a model that is
        collected later, e.g. out of a reference cycle, then has nothing left to destroy)."""
        if self.h:
            for m in list(self._models):
                m.close()
            lib().snnb_context_destroy(self.h)
            self.h = vp()

    def __del__(self):
        if sys.is_finalizing():  # interpreter shutdown: the CUDA runtime may already be gone, leave the handle to the OS
            return
        try:
            self.close()
        except Exception:
            pass


class ImageTexture:
    """Device tensor [N,H,W,C]; upload()/download() as in imageTexture.h, NHWC fp32 or the reference's C4HW4."""

    def __init__(self, ctx, n, h, w, c):
        self.ctx = ctx
        self.shape = (int(n), int(h), int(w), int(c))
        self.h = vp()
        check(lib().snnb_tensor_alloc(ctx.h, *self.shape, C.byref(self.h)), "snnb_tensor_alloc")

    @classmethod
    def from_numpy(cls, ctx, arr):
        arr = _f32(arr)
        assert arr.ndim == 4, "expect NHWC"
        t = cls(ctx, *arr.shape)
        t.upload(arr)
        return t

    def upload(self, arr):
        arr = _f32(arr)
        assert arr.shape == self.shape, (arr.shape, self.shape)
        check(lib().snnb_tensor_upload_nhwc(self.ctx.h, self.h, _ptr(arr)), "snnb_tensor_upload_nhwc")

    def download(self):
        out = np.empty(self.shape, dtype=np.float32)
        check(lib().snnb_tensor_download_nhwc(self.ctx.h, self.h, _ptr(out)), "snnb_tensor_download_nhwc")
        return out

    def upload_c4hw4(self, arr):
        n, h, w, c = self.shape
        arr = _f32(arr)
        assert arr.shape == (n, (c + 3) // 4, h, w, 4)
        check(lib().snnb_tensor_upload_c4hw4(self.ctx.h, self.h, _ptr(arr)), "snnb_tensor_upload_c4hw4")

    def download_c4hw4(self):
        n, h, w, c = self.shape
        out = np.empty((n, (c + 3) // 4, h, w, 4), dtype=np.float32)
        check(lib().snnb_tensor_download_c4hw4(self.ctx.h, self.h, _ptr(out)), "snnb_tensor_download_c4hw4")
        return out

    def dump(self, path):
        check(lib().snnb_tensor_dump(self.ctx.h, self.h, path.encode()), "snnb_tensor_dump")

    def free(self):
        if self.h:
            lib().snnb_tensor_free(self.h)
            self.h = vp()

    def __del__(self):
        if sys.is_finalizing():
            return
        try:
            self.free()
        except Exception:
            pass


class Weights:
    def __init__(self, handle):
        self.h = handle

    def free(self):
        if self.h:
            lib().snnb_weights_free(self.h)
            self.h = vp()

    def __del__(self):
        if sys.is_finalizing():
            return
        try:
            self.free()
        except Exception:
            pass


def conv_desc(ic, oc, k, stride=1, pad_x=0, pad_y=0, pad_mode="constant", activation="", alpha=0.0, algo="auto"):
    return ConvDesc(int(ic), int(oc), int(k), int(stride), int(pad_x), int(pad_y), PAD_MODE[pad_mode], ACT[activation], float(alpha), ALGO[algo])


def _bn_ptrs(bn):
    if bn is None:
        return [None] * 4, []
    keep = [_f32(bn[k]) for k in ("gamma", "beta", "mean", "var")]
    return [_ptr(a) for a in keep], keep


# ---- single-layer helpers (the boundary the reference's own op tests use: ShaderUnitTest::snn*TestWithLayer) ----
def conv2d(ctx, x, w_oihw, bias=None, bn=None, stride=1, pad_x=0, pad_y=0, pad_mode="constant", activation="", alpha=0.0, out_hw=None, residual=None,
           algo="auto"):
    x = _f32(x)
    w_oihw = _f32(w_oihw)
    n, h, w, ic = x.shape
    oc, ic2, k, _ = w_oihw.shape
    assert ic == ic2
    d = conv_desc(ic, oc, k, stride, pad_x, pad_y, pad_mode, activation, alpha, algo)
    bias_a = None if bias is None else _f32(bias)
    ptrs, keep = _bn_ptrs(bn)
    wh = vp()
    check(lib().snnb_weights_pack_conv2d(ctx.h, C.byref(d), _ptr(w_oihw), _ptr(bias_a), *ptrs, C.byref(wh)), "snnb_weights_pack_conv2d")
    wobj = Weights(wh)
    oh, ow = out_hw
    tin = ImageTexture.from_numpy(ctx, x)
    tout = ImageTexture(ctx, n, oh, ow, oc)
    tres = None if residual is None else ImageTexture.from_numpy(ctx, residual)
    check(lib().snnb_conv2d_launch(ctx.h, C.byref(d), wobj.h, tin.h, tres.h if tres else None, tout.h), "snnb_conv2d_launch")
    out = tout.download()
    del keep
    return out


def depthwise(ctx, x, w_chw, bias=None, bn=None, stride=1, pad_x=0, pad_y=0, activation="", alpha=0.0, out_hw=None):
    x = _f32(x)
    w_chw = _f32(w_chw)
    n, h, w, c = x.shape
    k = w_chw.shape[-1]
    d = conv_desc(c, c, k, stride, pad_x, pad_y, "constant", activation, alpha)
    bias_a = None if bias is None else _f32(bias)
    ptrs, keep = _bn_ptrs(bn)
    wh = vp()
    check(lib().snnb_weights_pack_depthwise(ctx.h, C.byref(d), _ptr(w_chw), _ptr(bias_a), *ptrs, C.byref(wh)), "snnb_weights_pack_depthwise")
    wobj = Weights(wh)
    oh, ow = out_hw
    tin = ImageTexture.from_numpy(ctx, x)
    tout = ImageTexture(ctx, n, oh, ow, c)
    check(lib().snnb_depthwise_launch(ctx.h, C.byref(d), wobj.h, tin.h, tout.h), "snnb_depthwise_launch")
    out = tout.download()
    del keep
    return out


def pool2d(ctx, x, k, stride, avg, out_hw):
    x = _f32(x)
    n, h, w, c = x.shape
    tin = ImageTexture.from_numpy(ctx, x)
    tout = ImageTexture(ctx, n, out_hw[0], out_hw[1], c)
    fn = lib().snnb_avgpool_launch if avg else lib().snnb_maxpool_launch
    check(fn(ctx.h, int(k), int(stride), tin.h, tout.h), "snnb_pool_launch")
    return tout.download()


def add(ctx, a, b, activation="", alpha=0.0):
    ta, tb = ImageTexture.from_numpy(ctx, a), ImageTexture.from_numpy(ctx, b)
    to = ImageTexture(ctx, *ta.shape)
    check(lib().snnb_add_launch(ctx.h, ACT[activation], float(alpha), ta.h, tb.h, to.h), "snnb_add_launch")
    return to.download()


def _channels(ctx, c, gamma=None, beta=None, mean=None, var=None):
    arrs = [None if a is None else _f32(a) for a in (gamma, beta, mean, var)]
    wh = vp()
    check(lib().snnb_weights_pack_channels(ctx.h, int(c), *[_ptr(a) for a in arrs], C.byref(wh)), "snnb_weights_pack_channels")
    return Weights(wh)


def batchnorm(ctx, x, bn, activation="", alpha=0.0):
    t = ImageTexture.from_numpy(ctx, x)
    w = _channels(ctx, t.shape[3], bn["gamma"], bn["beta"], bn["mean"], bn["var"])
    o = ImageTexture(ctx, *t.shape)
    check(lib().snnb_batchnorm_launch(ctx.h, w.h, ACT[activation], float(alpha), t.h, o.h), "snnb_batchnorm_launch")
    return o.download()


def instancenorm(ctx, x, gamma, beta, activation="", alpha=0.0):
    t = ImageTexture.from_numpy(ctx, x)
    w = _channels(ctx, t.shape[3], gamma, beta)
    o = ImageTexture(ctx, *t.shape)
    check(lib().snnb_instancenorm_launch(ctx.h, w.h, ACT[activation], float(alpha), t.h, o.h), "snnb_instancenorm_launch")
    return o.download()


def activation(ctx, x, activation, alpha=0.0):
    t = ImageTexture.from_numpy(ctx, x)
    o = ImageTexture(ctx, *t.shape)
    check(lib().snnb_activation_launch(ctx.h, ACT[activation], float(alpha), t.h, o.h), "snnb_activation_launch")
    return o.download()


def dense(ctx, x, kernel_out_in, bias=None, activation="", alpha=0.0):
    x = _f32(x)
    kernel_out_in = _f32(kernel_out_in)
    n_out, n_in = kernel_out_in.shape
    bias_a = None if bias is None else _f32(bias)
    wh = vp()
    check(lib().snnb_weights_pack_dense(ctx.h, n_in, n_out, _ptr(kernel_out_in), _ptr(bias_a), C.byref(wh)), "snnb_weights_pack_dense")
    w = Weights(wh)
    t = ImageTexture.from_numpy(ctx, x)
    o = ImageTexture(ctx, x.shape[0], 1, 1, n_out)
    check(lib().snnb_dense_launch(ctx.h, w.h, ACT[activation], float(alpha), t.h, o.h), "snnb_dense_launch")
    return o.download()


def softmax(ctx, x):
    t = ImageTexture.from_numpy(ctx, x)
    o = ImageTexture(ctx, *t.shape)
    check(lib().snnb_softmax_launch(ctx.h, t.h, o.h), "snnb_softmax_launch")
    return o.download()


def argmax1(ctx, x):
    t = ImageTexture.from_numpy(ctx, x)
    idx = (C.c_int * t.shape[0])()
    check(lib().snnb_argmax1(ctx.h, t.h, idx), "snnb_argmax1")
    return np.array(list(idx), dtype=np.int32)


def flatten(ctx, x):
    t = ImageTexture.from_numpy(ctx, x)
    n, h, w, c = t.shape
    o = ImageTexture(ctx, n, 1, 1, h * w * c)
    check(lib().snnb_flatten_launch(ctx.h, t.h, o.h), "snnb_flatten_launch")
    return o.download()


def concat(ctx, a, b):
    ta, tb = ImageTexture.from_numpy(ctx, a), ImageTexture.from_numpy(ctx, b)
    n, h, w, ca = ta.shape
    o = ImageTexture(ctx, n, h, w, ca + tb.shape[3])
    check(lib().snnb_concat_launch(ctx.h, ta.h, tb.h, o.h), "snnb_concat_launch")
    return o.download()


def upsample(ctx, x, scale, bilinear=False):
    t = ImageTexture.from_numpy(ctx, x)
    n, h, w, c = t.shape
    o = ImageTexture(ctx, n, int(h * scale), int(w * scale), c)
    check(lib().snnb_upsample_launch(ctx.h, float(scale), int(bool(bilinear)), t.h, o.h), "snnb_upsample_launch")
    return o.download()


def pad(ctx, x, pad_x, pad_y, out_hw, mode="constant"):
    t = ImageTexture.from_numpy(ctx, x)
    n, h, w, c = t.shape
    o = ImageTexture(ctx, n, out_hw[0], out_hw[1], c)
    check(lib().snnb_pad_launch(ctx.h, int(pad_x), int(pad_y), PAD_MODE[mode], t.h, o.h), "snnb_pad_launch")
    return o.download()


def subpixel(ctx, x, r):
    t = ImageTexture.from_numpy(ctx, x)
    n, h, w, c = t.shape
    o = ImageTexture(ctx, n, h * r, w * r, 1)
    check(lib().snnb_subpixel_launch(ctx.h, int(r), t.h, o.h), "snnb_subpixel_launch")
    return o.download()


class MixedInferenceCore:
    """snn::MixedInferenceCore: create(ctx, modelFileName, options) then run(images)."""

    def __init__(self, ctx, json_path, batch=1, input_hw=None, conv_algo="auto", use_cuda_graph=False, fuse=False, precision="fp32x3"):
        self.ctx = ctx
        self.batch = int(batch)
        opt = ModelOptions(self.batch, int(input_hw[1]) if input_hw else 0, int(input_hw[0]) if input_hw else 0, ALGO[conv_algo], int(bool(use_cuda_graph)),
                           int(bool(fuse)), PRECISION[precision])
        self.h = vp()
        check(lib().snnb_model_load_json(ctx.h, json_path.encode(), C.byref(opt), C.byref(self.h)), "snnb_model_load_json")
        ctx._models.add(self)

    @classmethod
    def create(cls, ctx, json_path, **kw):
        return cls(ctx, json_path, **kw)

    # -- introspection --
    @property
    def num_layers(self):
        return lib().snnb_model_num_layers(self.h)

    def layer_info(self, i):
        name = C.create_string_buffer(512)
        typ = C.create_string_buffer(64)
        d = [C.c_int() for _ in range(4)]
        check(lib().snnb_model_layer_info(self.h, i, name, 512, typ, 64, *[C.byref(v) for v in d]), "snnb_model_layer_info")
        return name.value.decode(), typ.value.decode(), tuple(v.value for v in d)

    def _dims(self, fn, idx):
        d = [C.c_int() for _ in range(4)]
        check(fn(self.h, idx, *[C.byref(v) for v in d]), "dims")
        return tuple(v.value for v in d)

    def input_shape(self, idx=0):
        return self._dims(lib().snnb_model_input_dims, idx)

    def output_shape(self, idx=0):
        return self._dims(lib().snnb_model_output_dims, idx)

    @property
    def num_inputs(self):
        return lib().snnb_model_num_inputs(self.h)

    @property
    def num_outputs(self):
        return lib().snnb_model_num_outputs(self.h)

    @property
    def launches_per_forward(self):
        return lib().snnb_model_launches_per_forward(self.h)

    # -- execution --
    def run(self, images, want_classes=True):
        """End to end with host buffers: returns (output0 NHWC fp32, 1-based class indices or None)."""
        images = _f32(images)
        assert images.shape == self.input_shape(0), (images.shape, self.input_shape(0))
        oshape = self.output_shape(0)
        out = np.empty(oshape, dtype=np.float32)
        classes = (C.c_int * self.batch)()
        check(lib().snnb_model_run(self.h, _ptr(images), _ptr(out), out.size, classes if want_classes else None), "snnb_model_run")
        return out, (np.array(list(classes), dtype=np.int32) if want_classes else None)

    def run_raw(self, in_ptr, out_ptr, out_floats, classes_ptr=None):
        """snnb_model_run on raw host addresses (pinned buffers owned by the caller, e.g. bench.py)."""
        check(lib().snnb_model_run(self.h, in_ptr, out_ptr, out_floats, classes_ptr), "snnb_model_run")

    def submit_raw(self, in_ptr, out_ptr, out_floats, classes_ptr=None):
        """snnb_model_submit on raw (pinned) host addresses; returns the ticket for wait()."""
        t = C.c_int()
        check(lib().snnb_model_submit(self.h, in_ptr, out_ptr, out_floats, classes_ptr, C.byref(t)), "snnb_model_submit")
        return t.value

    def submit_u8_raw(self, in_ptr, mean4, norm4, out_ptr, out_floats, classes_ptr=None):
        """snnb_model_submit_u8: 8-bit NHWC images, normalised on the device as (x - mean[c & 3]) * norm[c & 3]."""
        t = C.c_int()
        m = (C.c_float * 4)(*[float(v) for v in mean4])
        n = (C.c_float * 4)(*[float(v) for v in norm4])
        check(lib().snnb_model_submit_u8(self.h, in_ptr, m, n, out_ptr, out_floats, classes_ptr, C.byref(t)), "snnb_model_submit_u8")
        return t.value

    def run_u8(self, images_u8, mean4, norm4, want_classes=True):
        """Convenience wrapper: one batch of uint8 NHWC images through submit_u8 / wait (numpy in, numpy out)."""
        images_u8 = np.ascontiguousarray(images_u8, dtype=np.uint8)
        assert images_u8.shape == self.input_shape(0), (images_u8.shape, self.input_shape(0))
        out = np.empty(self.output_shape(0), np.float32)
        classes = (C.c_int * self.batch)() if want_classes else None
        t = self.submit_u8_raw(images_u8.ctypes.data, mean4, norm4, out.ctypes.data, out.size, classes)
        self.wait(t)
        return out, (np.array(list(classes), dtype=np.int32) if want_classes else None)

    def run_image(self, images_u8, mean4, norm4, linear=True, out_u8=False, out_scale=1.0, out_offset=0.0, want_classes=False):
        """snnb_model_submit_image + wait: u8 NHWC images of ANY size in (resized + normalised on the device), fp32 tensor or u8 image out."""
        from ._lib import ImageIO
        images_u8 = np.ascontiguousarray(images_u8, dtype=np.uint8)
        n, sh, sw, c = images_u8.shape
        oshape = self.output_shape(0)
        out = np.empty(oshape, np.uint8 if out_u8 else np.float32)
        classes = (C.c_int * self.batch)() if want_classes else None
        io = ImageIO()
        io.input_u8, io.src_height, io.src_width, io.linear_filter = images_u8.ctypes.data, sh, sw, int(bool(linear))
        io.mean4 = (C.c_float * 4)(*[float(v) for v in mean4])
        io.norm4 = (C.c_float * 4)(*[float(v) for v in norm4])
        io.output_capacity = out.size
        if out_u8:
            io.output_u8, io.out_scale, io.out_offset = out.ctypes.data, float(out_scale), float(out_offset)
        else:
            io.output_f32 = out.ctypes.data
        io.classes_1based = C.cast(classes, C.c_void_p) if want_classes else None
        t = C.c_int()
        check(lib().snnb_model_submit_image(self.h, C.byref(io), C.byref(t)), "snnb_model_submit_image")
        self.wait(t.value)
        return out, (np.array(list(classes), dtype=np.int32) if want_classes else None)

    def wait(self, ticket):
        check(lib().snnb_model_wait(self.h, int(ticket)), "snnb_model_wait")

    _TORCH_LAYOUTS = {"nhwc": _lib.LAYOUT_NHWC, "nchw": _lib.LAYOUT_NCHW}

    @staticmethod
    def _torch_dtypes():
        import torch
        return {torch.float32: _lib.DTYPE_F32, torch.float16: _lib.DTYPE_F16, torch.uint8: _lib.DTYPE_U8}

    @staticmethod
    def _nhwc_as(shape, layout):
        n, h, w, c = shape
        return (n, h, w, c) if layout == "nhwc" else (n, c, h, w)

    def _device_inputs(self, who, inputs, layout, mean4, norm4):
        """The snnb_device_buffer array for run_torch / detect_torch: returns (the contiguous tensors, which must stay alive until the
        call has enqueued its reads, the buffers)."""
        import torch
        dtypes = self._torch_dtypes()
        if layout not in self._TORCH_LAYOUTS:
            raise ValueError("%s: layout %r: expected 'nhwc' or 'nchw'" % (who, layout))
        xs = [inputs] if isinstance(inputs, torch.Tensor) else list(inputs)
        keep = [x.contiguous() for x in xs]  # the stream fence orders any reuse of the memory after the reads
        ins = (_lib.DeviceBuffer * max(1, len(keep)))()
        for i, x in enumerate(keep):
            if x.dtype not in dtypes:
                raise ValueError("%s: input %d has dtype %s; float32, float16 or uint8 is supported" % (who, i, x.dtype))
            want = self._nhwc_as(self.input_shape(i), layout) if i < self.num_inputs else None
            if want is not None and tuple(x.shape) != want:
                raise ValueError("%s: input %d has shape %s, the model takes %s (%s)" % (who, i, tuple(x.shape), want, layout))
            ins[i].data, ins[i].dtype, ins[i].layout = x.data_ptr(), dtypes[x.dtype], self._TORCH_LAYOUTS[layout]
            ins[i].mean4 = (C.c_float * 4)(*[float(v) for v in (mean4 if mean4 is not None else [0.0] * 4)])
            ins[i].norm4 = (C.c_float * 4)(*[float(v) for v in (norm4 if norm4 is not None else [1.0] * 4)])
        return keep, ins

    def _torch_stream(self):
        import torch
        # torch's default stream is the legacy NULL stream, which the library reads as "the context's stream": name it cudaStreamLegacy (1)
        return torch.cuda.current_stream(torch.device("cuda", self.ctx.device)).cuda_stream or 1

    def run_torch(self, inputs, layout="nhwc", mean4=None, norm4=None, out_dtype=None, out_layout="nhwc", out_scale=1.0, out_offset=0.0,
                  want_classes=False):
        """snnb_model_run_device with torch CUDA tensors, ordered on the current torch stream and never synchronising.

        inputs: a CUDA tensor (float32, float16 or uint8), or a list with one per model input, each batch x H x W x C ("nhwc") or
        batch x C x H x W ("nchw"); uint8 inputs are normalised as (x - mean4[c & 3]) * norm4[c & 3] (default mean 0, norm 1).
        Outputs are allocated here as out_dtype (float32 by default, float16 or uint8: clamp(round(v * out_scale + out_offset), 0, 255))
        in out_layout. Returns output 0 for a one-output model, else the list of outputs; with want_classes, (outputs, the 1-based
        classes as a device int32 tensor)."""
        if layout not in self._TORCH_LAYOUTS:
            raise ValueError("run_torch: layout %r: expected 'nhwc' or 'nchw'" % (layout,))
        outs, obufs, classes = self._device_outputs("run_torch", out_dtype, out_layout, out_scale, out_offset, want_classes)
        keep, ins = self._device_inputs("run_torch", inputs, layout, mean4, norm4)
        check(lib().snnb_model_run_device(self.h, ins, len(keep), obufs, len(outs), classes.data_ptr() if want_classes else None, self._torch_stream()),
              "snnb_model_run_device")
        result = outs[0] if len(outs) == 1 else outs
        return (result, classes) if want_classes else result

    def _device_outputs(self, who, out_dtype, out_layout, out_scale, out_offset, want_classes):
        """run_torch / run_frames: every model output allocated with torch as out_dtype in out_layout, their snnb_device_buffer array,
        and the classes tensor (or None)."""
        import torch
        dtypes, layouts = self._torch_dtypes(), self._TORCH_LAYOUTS
        out_dtype = torch.float32 if out_dtype is None else out_dtype
        if out_dtype not in dtypes or out_layout not in layouts:
            raise ValueError("%s: output dtype %s / layout %r: expected float32, float16 or uint8 and 'nhwc' or 'nchw'" % (who, out_dtype, out_layout))
        device = torch.device("cuda", self.ctx.device)
        outs = [torch.empty(self._nhwc_as(self.output_shape(j), out_layout), dtype=out_dtype, device=device) for j in range(self.num_outputs)]
        obufs = (_lib.DeviceBuffer * max(1, len(outs)))()
        for j, o in enumerate(outs):
            obufs[j].data, obufs[j].dtype, obufs[j].layout = o.data_ptr(), dtypes[out_dtype], layouts[out_layout]
            obufs[j].scale, obufs[j].offset = float(out_scale), float(out_offset)
        classes = torch.empty(self.batch, dtype=torch.int32, device=device) if want_classes else None
        return outs, obufs, classes

    def detect_torch(self, inputs, layout="nhwc", mean4=None, norm4=None, max_rows=100):
        """snnb_model_detect_device with torch CUDA tensors: the forward pass and the YOLO decode, score sort and NMS on the device,
        ordered on the current torch stream and never synchronising. Inputs as in run_torch.

        Returns (rows, counts): rows a CUDA float32 tensor batch x max_rows x 6 of {class, score, x, y, w, h}, zero past each image's
        count; counts a CUDA int32 tensor [batch] with min(kept boxes, max_rows, 100), the rows boxes(n) returns after run()."""
        import torch
        keep, ins = self._device_inputs("detect_torch", inputs, layout, mean4, norm4)
        device = torch.device("cuda", self.ctx.device)
        rows = torch.empty((self.batch, max(int(max_rows), 0), 6), dtype=torch.float32, device=device)
        counts = torch.empty(self.batch, dtype=torch.int32, device=device)
        check(lib().snnb_model_detect_device(self.h, ins, len(keep), rows.data_ptr() or None, int(max_rows), counts.data_ptr(), self._torch_stream()),
              "snnb_model_detect_device")
        return rows, counts

    _FRAME_FORMATS = {"nv12": _lib.FRAME_NV12, "nv21": _lib.FRAME_NV21, "i420": _lib.FRAME_I420, "rgba8": _lib.FRAME_RGBA8}
    _YUV_MATRICES = {"bt601": _lib.YUV_BT601, "bt709": _lib.YUV_BT709}

    def _frames(self, who, frames, format, matrix, linear, mean4, norm4):
        """The snnb_frames descriptor of a uint8 CUDA tensor: NV12 / NV21 / I420 as [N, H * 3 // 2, W] (the packed 4:2:0 layout, H and W
        even; NV12 / NV21 rows may be pitched, I420 rows must be dense), RGBA8 as [N, H, W, 4] (rows may be pitched). N is the batch."""
        f, n = self._frames_any(who, frames, format, matrix, linear, mean4, norm4)
        if n != self.batch:
            raise ValueError("%s: %d frames given, the model's batch is %d" % (who, n, self.batch))
        return f

    def _frames_any(self, who, frames, format, matrix, linear, mean4, norm4):
        """_frames for any number of frames: returns (the descriptor, the number of frames)."""
        if format not in self._FRAME_FORMATS or matrix not in self._YUV_MATRICES:
            raise ValueError("%s: format %r / matrix %r: expected one of %s and one of %s" % (who, format, matrix, sorted(self._FRAME_FORMATS),
                                                                                               sorted(self._YUV_MATRICES)))
        f = _lib.Frames()
        f.format, f.matrix, f.linear_filter = self._FRAME_FORMATS[format], self._YUV_MATRICES[matrix], int(bool(linear))
        f.mean4 = (C.c_float * 4)(*[float(v) for v in (mean4 if mean4 is not None else [0.0] * 4)])
        f.norm4 = (C.c_float * 4)(*[float(v) for v in (norm4 if norm4 is not None else [1.0] * 4)])
        return f, self._frame_planes(who, "frames", frames, format, f)

    @staticmethod
    def _frame_planes(who, what, frames, format, f):
        """The size, planes, pitches and image strides of an snnb_frames / snnb_frames_out `f` from a uint8 CUDA tensor in the layouts
        of _frames; returns the number of frames."""
        import torch
        if not isinstance(frames, torch.Tensor) or frames.dtype != torch.uint8:
            raise ValueError("%s: %s must be a uint8 CUDA tensor" % (who, what))
        shape, st, base = tuple(frames.shape), frames.stride(), frames.data_ptr()
        if format == "rgba8":
            if len(shape) != 4 or shape[3] != 4 or st[3] != 1 or st[2] != 4:
                raise ValueError("%s: rgba8 %s are [N, H, W, 4] with dense pixels; got shape %s, strides %s" % (who, what, shape, st))
            n, f.height, f.width = shape[0], shape[1], shape[2]
            f.plane[0], f.pitch[0], f.image_stride[0] = base, st[1], st[0]
        else:
            if len(shape) != 3 or shape[1] % 3 or shape[1] < 3 or shape[2] % 2 or st[2] != 1:
                raise ValueError("%s: %s %s are [N, H * 3 // 2, W] with H and W even and dense rows; got shape %s, strides %s" % (who, format, what, shape, st))
            n, f.height, f.width = shape[0], shape[1] // 3 * 2, shape[2]
            pitch = st[1]
            if format == "i420" and pitch != f.width:
                raise ValueError("%s: i420 %s must have dense rows (row stride %d, width %d)" % (who, what, pitch, f.width))
            f.plane[0], f.pitch[0] = base, pitch
            f.plane[1], f.pitch[1] = base + f.height * pitch, pitch if format != "i420" else f.width // 2
            if format == "i420":
                f.plane[2], f.pitch[2] = base + f.height * pitch + (f.height // 2) * (f.width // 2), f.width // 2
            for p in range(3):
                f.image_stride[p] = st[0]
        return n

    def run_frames(self, frames, format="nv12", matrix="bt601", linear=True, mean4=None, norm4=None, out_dtype=None, out_layout="nhwc", out_scale=1.0,
                   out_offset=0.0, want_classes=False):
        """snnb_model_run_frames: a batch of 8-bit video frames of any size on the GPU (NV12, NV21, I420 or RGBA8, see _frames) converted
        to RGBA8 exactly as libyuv does, resized to the model input (linear or nearest, as run_image), normalised as
        (x - mean4[c]) * norm4[c] (default mean 0, norm 1) and run, ordered on the current torch stream and never synchronising.
        Model channel c is RGBA component c. Outputs and classes as run_torch."""
        outs, obufs, classes = self._device_outputs("run_frames", out_dtype, out_layout, out_scale, out_offset, want_classes)
        f = self._frames("run_frames", frames, format, matrix, linear, mean4, norm4)
        check(lib().snnb_model_run_frames(self.h, C.byref(f), obufs, len(outs), classes.data_ptr() if want_classes else None, self._torch_stream()),
              "snnb_model_run_frames")
        result = outs[0] if len(outs) == 1 else outs
        return (result, classes) if want_classes else result

    def run_rois(self, frames, rois, count=None, format="nv12", matrix="bt601", linear=True, mean4=None, norm4=None, out_dtype=None, out_layout="nhwc",
                 out_scale=1.0, out_offset=0.0, want_classes=False):
        """snnb_model_run_rois: regions of device frames as the batch. frames: any number of frames in _frames' layouts. rois: an int32
        CUDA tensor [batch, 6] of {frame, row, x, y, width, height} (rois_from_detections makes one); count: None (every slot is used)
        or an int32 CUDA tensor of one element (slots i < clamp(count, 0, batch) are used). Each used slot whose region lies inside an
        existing frame gets exactly what run_frames computes for that region cut out as an RGBA8 frame of its own; every other slot
        comes out all zero, class 0. Outputs, classes and the stream contract as run_frames."""
        import torch
        if not (isinstance(rois, torch.Tensor) and rois.is_cuda and rois.dtype == torch.int32 and tuple(rois.shape) == (self.batch, 6)):
            raise ValueError("run_rois: rois must be an int32 CUDA tensor [%d, 6] (the model's batch)" % self.batch)
        if count is not None and not (isinstance(count, torch.Tensor) and count.is_cuda and count.dtype == torch.int32 and count.numel() == 1):
            raise ValueError("run_rois: count must be None or an int32 CUDA tensor of one element")
        outs, obufs, classes = self._device_outputs("run_rois", out_dtype, out_layout, out_scale, out_offset, want_classes)
        f, n = self._frames_any("run_rois", frames, format, matrix, linear, mean4, norm4)
        rois = rois.contiguous()
        check(lib().snnb_model_run_rois(self.h, C.byref(f), n, rois.data_ptr(), count.data_ptr() if count is not None else None, obufs, len(outs),
                                        classes.data_ptr() if want_classes else None, self._torch_stream()),
              "snnb_model_run_rois")
        result = outs[0] if len(outs) == 1 else outs
        return (result, classes) if want_classes else result

    def detect_frames(self, frames, format="nv12", matrix="bt601", linear=True, mean4=None, norm4=None, max_rows=100):
        """snnb_model_detect_frames: run_frames' input, detect_torch's forward pass, device decode and (rows, counts)."""
        import torch
        f = self._frames("detect_frames", frames, format, matrix, linear, mean4, norm4)
        device = torch.device("cuda", self.ctx.device)
        rows = torch.empty((self.batch, max(int(max_rows), 0), 6), dtype=torch.float32, device=device)
        counts = torch.empty(self.batch, dtype=torch.int32, device=device)
        check(lib().snnb_model_detect_frames(self.h, C.byref(f), rows.data_ptr() or None, int(max_rows), counts.data_ptr(), self._torch_stream()),
              "snnb_model_detect_frames")
        return rows, counts

    def transform_frames(self, frames, format="nv12", matrix="bt601", linear=True, mean4=None, norm4=None, out_format=None, out_hw=None,
                         out_linear=True, out_scale=1.0, out_offset=0.0, out=None):
        """snnb_model_transform_frames: run_frames' input and forward pass, then output 0 (1, 3 or 4 channels) written as 8-bit frames:
        clamp(round(v * out_scale + out_offset), 0, 255) as RGBA8 (1 channel: grey; 3: alpha 255), resized to out_hw (linear or
        nearest, as run_image) and converted as libyuv's ABGRToNV12 / ABGRToNV21 / ABGRToI420 (BT.601 limited range). Ordered on the
        current torch stream and never synchronising.

        out_format defaults to `format` and out_hw to the input frames' size. Returns `out`, a uint8 CUDA tensor in _frames' layouts
        ([N, H * 3 // 2, W] for the YUV formats, [N, H, W, 4] for RGBA8), allocated here unless given; it may be `frames` itself."""
        import torch
        out_format = format if out_format is None else out_format
        if out_format not in self._FRAME_FORMATS:
            raise ValueError("transform_frames: out_format %r: expected one of %s" % (out_format, sorted(self._FRAME_FORMATS)))
        f = self._frames("transform_frames", frames, format, matrix, linear, mean4, norm4)
        oh, ow = (f.height, f.width) if out_hw is None else (int(out_hw[0]), int(out_hw[1]))
        if out is None:
            if out_format != "rgba8" and (oh % 2 or ow % 2):
                raise ValueError("transform_frames: %s frames of %d x %d: the packed layout needs H and W even" % (out_format, oh, ow))
            shape = (self.batch, oh, ow, 4) if out_format == "rgba8" else (self.batch, oh * 3 // 2, ow)
            out = torch.empty(shape, dtype=torch.uint8, device=torch.device("cuda", self.ctx.device))
        o = _lib.FramesOut()
        o.format, o.linear_filter, o.scale, o.offset = self._FRAME_FORMATS[out_format], int(bool(out_linear)), float(out_scale), float(out_offset)
        n = self._frame_planes("transform_frames", "out frames", out, out_format, o)
        if n != self.batch or (out_hw is not None and (o.height, o.width) != (oh, ow)):
            raise ValueError("transform_frames: out holds %d frames of %d x %d; expected %d of %d x %d" % (n, o.height, o.width, self.batch, oh, ow))
        check(lib().snnb_model_transform_frames(self.h, C.byref(f), C.byref(o), self._torch_stream()), "snnb_model_transform_frames")
        return out

    def transform_luma(self, frames, format="nv12", linear=True, mean=0.0, norm=1.0, out_format=None, out_hw=None, out_linear=True, out_scale=1.0,
                       out_offset=0.0, out=None):
        """snnb_model_transform_luma, for a model with one 1-channel input and a 1-channel output 0 (ESPCN-style super-resolution, a
        luma denoiser): the Y plane of NV12 / NV21 / I420 frames, resized to the model input (linear or nearest, as run_image) and
        normalised as (Y - mean) * norm, feeds the model; clamp(round(v * out_scale + out_offset), 0, 255) of output 0, resized to out_hw
        (out_linear), is written as the Y plane of `out`, and the source U and V planes are resized plane to plane beside it. No colour
        conversion happens. Ordered on the current torch stream and never synchronising.

        A model trained on Y / 255 of full-range luma takes mean=0, norm=1/255 and gives back out_scale=255. Decoder frames are usually
        limited range, Y in [16, 235]: that model then takes mean=16, norm=1/219, and out_scale=219, out_offset=16 write its output
        back in the decoder's range.

        out_format defaults to `format` and out_hw to the input frames' size. Returns `out`, a uint8 CUDA tensor [N, H * 3 // 2, W] in
        _frames' layouts, allocated here unless given; it may be `frames` itself (same format and size), for an in-place filter."""
        import torch
        out_format = format if out_format is None else out_format
        if format not in self._FRAME_FORMATS or out_format not in self._FRAME_FORMATS:
            raise ValueError("transform_luma: format %r / out_format %r: expected one of %s" % (format, out_format, sorted(self._FRAME_FORMATS)))
        f = self._frames("transform_luma", frames, format, "bt601", linear, [float(mean)] * 4, [float(norm)] * 4)
        oh, ow = (f.height, f.width) if out_hw is None else (int(out_hw[0]), int(out_hw[1]))
        if out is None:
            if out_format == "rgba8":
                raise ValueError("transform_luma: out_format 'rgba8' has no Y plane; expected nv12, nv21 or i420")
            if oh % 2 or ow % 2:
                raise ValueError("transform_luma: %s frames of %d x %d: the packed layout needs H and W even" % (out_format, oh, ow))
            out = torch.empty((self.batch, oh * 3 // 2, ow), dtype=torch.uint8, device=torch.device("cuda", self.ctx.device))
        o = _lib.FramesOut()
        o.format, o.linear_filter, o.scale, o.offset = self._FRAME_FORMATS[out_format], int(bool(out_linear)), float(out_scale), float(out_offset)
        n = self._frame_planes("transform_luma", "out frames", out, out_format, o)
        if n != self.batch or (out_hw is not None and (o.height, o.width) != (oh, ow)):
            raise ValueError("transform_luma: out holds %d frames of %d x %d; expected %d of %d x %d" % (n, o.height, o.width, self.batch, oh, ow))
        check(lib().snnb_model_transform_luma(self.h, C.byref(f), C.byref(o), self._torch_stream()), "snnb_model_transform_luma")
        return out

    def segment_frames(self, frames, format="nv12", matrix="bt601", linear=True, mean4=None, norm4=None, luma=False, out_hw=None, out_linear=True,
                       threshold=0.5, out=None):
        """snnb_model_segment_frames, for segmentation models: run_frames' input and forward pass (luma=True: the Y plane into a
        1-channel input, as transform_luma feeds it), then the class scores of output 0 resized to out_hw (out_linear: bilinear, else
        nearest, with run_image's taps, on the fp32 scores) and reduced to one label byte per pixel: the arg-max over the channels
        (ties to the lowest index, NaN never wins, all NaN gives 0), or for a 1-channel output 1 where the score is >= threshold.
        Ordered on the current torch stream and never synchronising.

        out_hw defaults to the input frames' size. Returns `out`, a uint8 CUDA tensor [N, H, W] with dense pixels, allocated here
        unless given; a given `out` may have a row stride larger than W and any image stride."""
        import torch
        f = self._frames("segment_frames", frames, format, matrix, linear, mean4, norm4)
        oh, ow = (f.height, f.width) if out_hw is None else (int(out_hw[0]), int(out_hw[1]))
        if out is None:
            out = torch.empty((self.batch, oh, ow), dtype=torch.uint8, device=torch.device("cuda", self.ctx.device))
        if not (isinstance(out, torch.Tensor) and out.dtype == torch.uint8 and out.dim() == 3 and out.stride(2) == 1):
            raise ValueError("segment_frames: out must be a uint8 CUDA tensor [N, H, W] with dense pixels")
        if out.shape[0] != self.batch or (out_hw is not None and tuple(out.shape[1:]) != (oh, ow)):
            raise ValueError("segment_frames: out holds %d planes of %d x %d; expected %d of %d x %d" % (out.shape[0], out.shape[1], out.shape[2],
                                                                                                       self.batch, oh, ow))
        o = _lib.LabelsOut()
        o.height, o.width, o.plane = out.shape[1], out.shape[2], out.data_ptr()
        o.pitch, o.image_stride = out.stride(1), out.stride(0)
        o.linear_filter, o.threshold = int(bool(out_linear)), float(threshold)
        check(lib().snnb_model_segment_frames(self.h, C.byref(f), int(bool(luma)), C.byref(o), self._torch_stream()), "snnb_model_segment_frames")
        return out

    def set_input(self, images, idx=0):
        images = _f32(images)
        check(lib().snnb_model_set_input(self.h, idx, _ptr(images)), "snnb_model_set_input")
        self.ctx.sync()

    def forward(self):
        check(lib().snnb_model_forward(self.h), "snnb_model_forward")

    def get_output(self, idx=0):
        out = np.empty(self.output_shape(idx), dtype=np.float32)
        check(lib().snnb_model_get_output(self.h, idx, _ptr(out), out.size), "snnb_model_get_output")
        return out

    def layer_output(self, layer):
        _, _, shape = self.layer_info(layer)
        out = np.empty(shape, dtype=np.float32)
        check(lib().snnb_model_layer_output(self.h, layer, _ptr(out), out.size), "snnb_model_layer_output")
        return out

    def time_layers(self):
        n = self.num_layers
        arr = (C.c_float * n)()
        check(lib().snnb_model_time_layers(self.h, arr, n), "snnb_model_time_layers")
        return np.array(list(arr), dtype=np.float32)

    def layer_kernel(self, layer):
        """Kernel launched by `layer` in the last time_layers() pass ("" if none)."""
        buf = C.create_string_buffer(128)
        check(lib().snnb_model_layer_kernel(self.h, int(layer), buf, 128), "snnb_model_layer_kernel")
        return buf.value.decode()

    def dump_outputs(self, directory):
        check(lib().snnb_model_dump_outputs(self.h, directory.encode()), "snnb_model_dump_outputs")

    def boxes(self, n=0, max_rows=100):
        rows = (C.c_float * (6 * max_rows))()
        cnt = C.c_int()
        check(lib().snnb_model_get_boxes(self.h, n, rows, max_rows, C.byref(cnt)), "snnb_model_get_boxes")
        return np.array(list(rows), dtype=np.float32).reshape(max_rows, 6)[:cnt.value]

    def weight_arena(self):
        p = vp()
        b = C.c_size_t()
        check(lib().snnb_model_weight_arena(self.h, C.byref(p), C.byref(b)), "snnb_model_weight_arena")
        return p.value, b.value

    def close(self):
        if self.h:
            lib().snnb_model_destroy(self.h)
            self.h = vp()

    def __del__(self):
        if sys.is_finalizing():  # interpreter shutdown: the CUDA runtime may already be gone, leave the handle to the OS
            return
        try:
            self.close()
        except Exception:
            pass
