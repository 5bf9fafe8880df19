"""Device-resident inputs and outputs (snnb_model_run_device through MixedInferenceCore.run_torch) against the host paths, on one GPU.

    python tools/device_io_bench.py --out DIR [--seconds 2] [--rounds 3]

Writes DIR/device_io_bench.json and prints it. Four parts by default, and opt-in ones (see --parts; p010 compares 10-bit frames with
NV12 on detect_frames, transform_luma and transform_frames, with each frame kernel's time and bytes/s), all in one process:

  throughput   ResNet-18 224x224 batch 32 fed with uint8 NCHW images already on the GPU (what a GPU JPEG decoder returns), device
               classes and logits out, against snnb_model_submit_u8 / snnb_model_wait from pinned host uint8 NHWC images; and Candy 720x720
               batch 8, uint8 NCHW in and uint8 NCHW out, against snnb_model_submit_image / wait with pinned host uint8 in and out. The two
               paths alternate, `rounds` times, each for at least `seconds` after warm-up; frames/s = images over host time ending in a
               device synchronise.
  conversions  each conversion kernel's device time, from torch.profiler (CUDA activity) over 50 calls per configuration in a run of its
               own, and bytes read + written (from shapes) over that time against the H100 SXM's 3.35 TB/s of HBM3: the kernels do no
               arithmetic to speak of, so HBM bandwidth is their bound. A 64-channel tensor compares NCHW with NHWC, the case where the
               tensor-side accesses of NCHW threads are strided.
  detector     YOLOv3-tiny 416x416 batch 16: uint8 NCHW CUDA frames into detect_torch (decode, score sort and NMS on the device, boxes
               in device memory) against snnb_model_submit_u8 / wait + snnb_model_get_boxes for every image from pinned host memory,
               alternating as above; and the device time of the decode kernels (yolo_select / yolo_rank / yolo_nms) next to the forward
               pass's kernels, from torch.profiler over 50 calls, on the synthetic heads and on all-pass heads (every cell passes).
  frames       YOLOv3-tiny 416x416 batch 16 and ResNet-18 224x224 batch 32 fed with 1920x1080 NV12 frames on the GPU (what NVDEC
               returns): detect_frames / run_frames (colour conversion, resize and normalisation in frame_input_kernel) against what a
               user does without them, a torch NV12 -> RGB conversion (BT.601 limited range, float) + F.interpolate (bilinear) + the
               normalisation, then detect_torch / run_torch with the float32 NCHW tensor; alternating as above. And frame_input_kernel's
               device time per batch from torch.profiler over 50 calls, with bytes/s from what it must move: the model-input planes it
               writes, plus the source bytes under its taps (4 per output pixel, each a Y byte and a UV pair, capped by the planes'
               sizes), or plus the whole frame as the upper bound.
  transform    (opt-in) Candy 720x720 batch 8 from 1920x1080 NV12 frames to 1920x1080 NV12 frames: transform_frames (output 0 resized
               and converted to NV12 in frame_output_kernel) against what a user does without it, run_frames(out_dtype=uint8) then
               F.interpolate (bilinear), a torch RGB -> NV12 conversion (BT.601 limited range) and packing; alternating as above. And
               frame_output_kernel's device time per batch from torch.profiler over 50 calls, with bytes/s from the frame planes it writes
               plus the model-output planes it reads under its taps.
  rois         (opt-in) The second stage of a detection pipeline on 1920x1080 NV12 frames. (a) The full chain: YOLOv3-tiny 416x416
               batch 16 with all-pass heads (every cell passes, so each frame has 100 rows and the second stage always gets its 64
               regions) detect_frames -> rois_from_detections -> ResNet-18 112x112 batch 64 run_rois, against what a user does without
               them: rows and counts to the host, a torch NV12 -> RGB conversion, a crop + F.interpolate (bilinear) per box, stack,
               normalise, then run_torch; frames/s are detector frames, alternating as above. (b) The input kernel alone on a fixed grid
               of caller-made regions (2 x 2 cells of 960x540 in each of the 16 frames: 64 regions): frame_roi_input_kernel's device
               time per batch from torch.profiler over 50 calls, with bytes/s from the model-input planes it writes plus the source bytes
               under its taps (4 per model pixel, each a Y byte and a UV pair, capped by the region's size).
  luma         (opt-in) ESPCN at 1920x1080 (the size of the reference's runESPCN input), batch 1 and 4, from 1920x1080 NV12 frames
               to 3840x2160 NV12 frames: transform_luma (the Y plane into the model, output 0 out as the Y plane, U and V resized in
               luma_output_kernel) against what a user does without it, the Y plane made dense, run_torch with uint8 in and out,
               F.interpolate (bilinear) of U and V and packing; alternating as above. And the device time per batch of the input kernel
               (frame_input_kernel<luma>) and of luma_output_kernel from torch.profiler over 50 calls, with bytes/s from what each moves.
  segment      (opt-in) The U-Net of the model zoo at 256x256 x 1, batch 8, with 1 class (the reference's graph) and with 21, from
               1920x1080 NV12 frames (run_frames' input, both paths) to 1920x1080 label planes: segment_frames (scores resampled and reduced
               in segment_output_kernel) against what a user does without it, run_frames(out_dtype=float32) + F.interpolate (bilinear) +
               the arg-max (or the 0.5 threshold) + .to(uint8); alternating as above. And segment_output_kernel's time per batch from
               CUDA events (segment_frames calls less calls that run only the same input and forward pass) and from torch.profiler, with
               bytes/s from the labels written plus the model-output planes read once.
  framelist   (opt-in) Sixteen streams of mixed sizes, each frame its own allocation (4 x 3840x2160, 8 x 1920x1080, 4 x 1280x720 NV12):
               YOLOv3-tiny 416x416 batch 16 with all-pass heads detect_frame_list -> rois_from_detections with per-frame sizes ->
               ResNet-18 112x112 batch 64 run_rois_list, against what a user does without frame lists: per frame a torch NV12 -> RGB
               conversion and F.interpolate into one batch, detect_torch, rows to the host, crops as in `rois`, run_torch; alternating
               as above. The device time of each kernel of the chain from torch.profiler over 50 calls, and frame_input_kernel's list
               form against its batch form on one uniform 1920x1080 batch of 16 (the cost of the per-image descriptor).
  framelist_out (opt-in) The same sixteen streams written back: Candy 720x720 transform_frame_list in place, ESPCN 540x960 (the
               luma part's model at a quarter of the area, so that a batch of 16 fits) transform_luma_list in place, and the U-Net of
               `segment` (21 classes) segment_frame_list to each stream's size; each against what a user does without output lists,
               run_frame_list with a U8 (labels: float32) output, then per stream a torch resize, conversion and pack into that stream's
               frame (luma: each Y plane resized into one batch for run_torch, and back). And each list output kernel's device time
               from torch.profiler over 50 calls against its batch kernel on one uniform 1920x1080 list of 16.
  partial     (opt-in) Partial batches. ResNet-18 224x224 loaded at 32, run_torch (uint8 in, float32 out, device classes) at n = 1, 2, 4,
               8, 16 and 32 images: the batch-32 model after set_batch(n), a model loaded at batch n, and the batch-32 model fed 32 images
               of which n are used. And the `framelist` chain when only k = 4, 8, 12 or 16 of its streams have a frame:
               detect_frame_list on the batch-16 detector after set_batch(k), against the list padded to 16 with the k frames repeated.
               Frames/s count the frames a call needs; alternating as above.
  counted     (opt-in) Count-sized region batches. ResNet-18 112x112 loaded at 64 with sizes [8, 16, 32] declared, fed the 64 caller-made
               regions of `rois` (b) with a device-side count k = 0 .. 64: run_rois against the same call on a handle with no sizes declared
               and against a third handle after set_batch(bucket(k)), the size k selects; calls/s and the regions/s of the k used slots,
               alternating as above. And the `framelist` chain with planted detector heads and a min_score that keeps about three boxes per
               frame, four frame sets in turn, with and without sizes declared; the count of each frame set is reported beside the rates.
  tiled       (opt-in) Detection on tiles of 4 x 3840x2160 NV12 frames: each frame cut by snnb_tile_rois into 960x960 tiles with at
               least 96 px of overlap (5 x 3 = 15) plus one whole-frame region, 64 slots into YOLOv3-tiny 416x416 loaded at 64, with
               planted heads (scores scattered around 0.35) and with all-pass heads. (a) detect_rois; (b) what a user does without it,
               a torch NV12 -> RGB conversion, a crop + F.interpolate (bilinear) per tile, detect_torch, the rows to the host and
               tests/_region_merge.py's merge_region_rows in numpy; (c) detect_frames on the 4 frames alone (the price of tiling). Frames/s
               alternating as above (one warm-up call each: (b)'s merge takes seconds with all-pass heads). And, from torch.profiler
               in a run of its own, the merge kernels' device time per call against the whole call's.
  card        name, power limit and maximum SM clock, read by nvidia-smi in the same run.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    name, power, clock = [s.strip() for s in q.stdout.strip().split(",")] if q.returncode == 0 else ("?", "?", "?")
    return {"name": name, "power_limit": power, "sm_clock_max": clock}


def timed(fn, seconds, batch, sync):
    """Call fn() until `seconds` have passed; frames/s over the host time of the calls plus the final synchronise."""
    n, t0 = 0, time.perf_counter()
    while True:
        fn()
        n += 1
        if n % 8 == 0 and time.perf_counter() - t0 >= seconds:
            break
    sync()
    dt = time.perf_counter() - t0
    return {"frames_per_s": n * batch / dt, "calls": n, "seconds": dt}


class HostPipeline:
    """Double-buffered snnb_model_submit_u8 / submit_image + wait from pinned host buffers (bench.py's e2e loop)."""

    def __init__(self, torch, m, images_u8_nhwc, mean4, norm4, image_out):
        from shadernn_b200._lib import ImageIO
        self.m, self.image_out, self.mean4, self.norm4 = m, image_out, mean4, norm4
        self.ins = [torch.from_numpy(images_u8_nhwc).pin_memory() for _ in range(2)]
        n_out = int(np.prod(m.output_shape(0)))
        self.outs = [torch.empty(n_out, dtype=torch.uint8 if image_out else torch.float32).pin_memory() for _ in range(2)]
        self.cls = [torch.zeros(m.batch, dtype=torch.int32).pin_memory() for _ in range(2)]
        self.io = []
        for i in range(2):
            io = ImageIO()
            _, h, w, _ = images_u8_nhwc.shape
            io.input_u8, io.src_height, io.src_width, io.linear_filter = self.ins[i].data_ptr(), h, w, 1
            io.mean4, io.norm4 = (C.c_float * 4)(*mean4), (C.c_float * 4)(*norm4)
            io.output_u8, io.output_capacity, io.out_scale, io.out_offset = self.outs[i].data_ptr(), n_out, 1.0, 0.0
            self.io.append(io)
        self.pending, self.i = None, 0

    def step(self):
        from shadernn_b200._lib import check, lib
        k = self.i & 1
        if self.image_out:
            t = C.c_int()
            check(lib().snnb_model_submit_image(self.m.h, C.byref(self.io[k]), C.byref(t)), "snnb_model_submit_image")
            t = t.value
        else:
            t = self.m.submit_u8_raw(self.ins[k].data_ptr(), self.mean4, self.norm4, self.outs[k].data_ptr(), self.outs[k].numel(), self.cls[k].data_ptr())
        if self.pending is not None:
            self.m.wait(self.pending)
        self.pending, self.i = t, self.i + 1

    def drain(self):
        if self.pending is not None:
            self.m.wait(self.pending)
            self.pending = None


def throughput(torch, ctx, core, modelzoo, d, args):
    res = {}
    cases = [("resnet18", (224, 224), 32, ([127.5] * 4, [1.0 / 127.5] * 4), False), ("candy", (720, 720), 8, ([0.0] * 4, [1.0] * 4), True)]
    for name, hw, batch, (mean4, norm4), image_out in cases:
        path, _ = modelzoo.build(name, os.path.join(d, name), input_hw=hw)
        m = core.MixedInferenceCore(ctx, path, batch=batch, input_hw=hw, fuse=True, use_cuda_graph=True)
        img = np.random.default_rng(1).integers(0, 256, (batch, hw[0], hw[1], 3), dtype=np.uint8)
        dev_in = torch.from_numpy(img.transpose(0, 3, 1, 2).copy()).cuda()
        if image_out:
            dev = lambda: m.run_torch(dev_in, layout="nchw", mean4=mean4, norm4=norm4, out_dtype=torch.uint8, out_layout="nchw")  # noqa: E731
        else:
            dev = lambda: m.run_torch(dev_in, layout="nchw", mean4=mean4, norm4=norm4, want_classes=True)  # noqa: E731
        hp = HostPipeline(torch, m, img, mean4, norm4, image_out)
        for _ in range(5):
            dev()
            hp.step()
        hp.drain()
        torch.cuda.synchronize()
        rounds = []
        for _ in range(args.rounds):
            r_dev = timed(dev, args.seconds, batch, torch.cuda.synchronize)
            r_host = timed(hp.step, args.seconds, batch, hp.drain)
            rounds.append({"device": r_dev, "host": r_host})
        med = lambda k: float(np.median([r[k]["frames_per_s"] for r in rounds]))  # noqa: E731
        res[name] = {
            "shape": "%dx%d batch %d" % (hw[0], hw[1], batch),
            "device_path": "run_torch: uint8 NCHW CUDA tensor in, " + ("uint8 NCHW CUDA tensor out" if image_out else "fp32 logits + int32 classes as CUDA tensors out"),
            "host_path": ("snnb_model_submit_image/wait: pinned uint8 NHWC in, pinned uint8 NHWC out" if image_out else
                          "snnb_model_submit_u8/wait: pinned uint8 NHWC in, pinned fp32 logits + classes out"),
            "device_frames_per_s_median": med("device"),
            "host_frames_per_s_median": med("host"),
            "device_over_host": med("device") / med("host"),
            "rounds": rounds,
        }
        m.close()
    return res


def kernel_times_us(torch, fn, calls):
    """Average device time (us) per launch of the input and the output conversion kernel fn() launches (device_input*_kernel,
    device_output_kernel)."""
    from torch.profiler import ProfilerActivity, profile
    for _ in range(5):
        fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        if "snnb::device_input" in e.key or "snnb::device_output" in e.key:
            total = getattr(e, "device_time_total", None)
            total = e.cuda_time_total if total is None else total
            kind = "input" if "snnb::device_input" in e.key else "output"
            out[kind] = {"kernel": e.key, "launches": e.count, "us_per_launch": total / e.count}
    return out


def conversions(torch, ctx, core, modelzoo, d, calls=50):
    res = []
    # (label, model, hw, batch, input dtype, input layout, output dtype, output layout, bytes read + written per pixel by the input kernel
    # and by the output kernel). The tensor side is split-fp16: 2 planes x 2 bytes x Cp (= C rounded up to 8) per pixel; ResNet-18's input
    # is read by its stem alone, so only the 4-channel feed copy is written (2 planes x 2 bytes x 4).
    b = modelzoo.Builder()
    b.batchnorm(b.input(112, 112, 64))
    wide = modelzoo.write_model(b.layers, os.path.join(d, "bn64.json"))
    cases = [
        ("resnet18 u8 nchw in (feed copy only)", "resnet18", (224, 224), 32, torch.uint8, "nchw", None, None, 3 * 1 + 16, None),
        ("candy u8 nchw in / u8 nchw out", "candy", (720, 720), 8, torch.uint8, "nchw", torch.uint8, "nchw", 3 * 1 + 32, 32 + 3 * 1),
        ("candy f32 nhwc in / f32 nhwc out", "candy", (720, 720), 8, torch.float32, "nhwc", torch.float32, "nhwc", 3 * 4 + 32, 32 + 3 * 4),
        ("64 channels f32 nhwc in / out", wide, (112, 112), 32, torch.float32, "nhwc", torch.float32, "nhwc", 64 * 4 + 64 * 4, 64 * 4 + 64 * 4),
        ("64 channels f32 nchw in / out", wide, (112, 112), 32, torch.float32, "nchw", torch.float32, "nchw", 64 * 4 + 64 * 4, 64 * 4 + 64 * 4),
        ("64 channels f16 nchw in / out", wide, (112, 112), 32, torch.float16, "nchw", torch.float16, "nchw", 64 * 2 + 64 * 4, 64 * 4 + 64 * 2),
    ]
    paths = {}
    for label, name, hw, batch, din, lin, dout, lout, in_bpp, out_bpp in cases:
        if name.endswith(".json"):
            path = name
        else:
            if (name, hw) not in paths:
                paths[(name, hw)], _ = modelzoo.build(name, os.path.join(d, "%s_%d" % (name, hw[0])), input_hw=hw)
            path = paths[(name, hw)]
        m = core.MixedInferenceCore(ctx, path, batch=batch, input_hw=hw, fuse=True, use_cuda_graph=True)
        n, h, w, c = m.input_shape(0)
        shape = (n, h, w, c) if lin == "nhwc" else (n, c, h, w)
        x = (torch.randint(0, 256, shape, dtype=torch.uint8) if din == torch.uint8 else torch.rand(shape).to(din)).cuda()
        kw = {"layout": lin}
        if dout is not None:
            kw.update(out_dtype=dout, out_layout=lout)
        times = kernel_times_us(torch, lambda: m.run_torch(x, **kw), calls)
        px = n * h * w
        for kind, bpp in (("input", in_bpp), ("output", out_bpp)):
            if bpp is None or kind not in times:
                continue
            t = times[kind]
            nbytes = px * bpp
            t.update({"case": label, "bytes": nbytes, "bytes_per_s": nbytes / (t["us_per_launch"] * 1e-6)})
            t["share_of_hbm_peak"] = t["bytes_per_s"] / HBM_BYTES_PER_S
            t["bound"] = "HBM bandwidth (3.35 TB/s, H100 SXM data sheet)"
            res.append(t)
        m.close()
    return res


def detector_kernel_times_us(torch, fn, calls):
    """Device time per call (us) of the decode kernels, the forward pass's kernels and the input conversion that fn() launches."""
    from torch.profiler import ProfilerActivity, profile
    for _ in range(5):
        fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            fn()
        torch.cuda.synchronize()
    out = {"decode": {}, "forward_us": 0.0, "input_us": 0.0}
    for e in prof.key_averages():
        total = getattr(e, "device_time_total", None)
        total = e.cuda_time_total if total is None else total
        if "snnb::" not in e.key or total <= 0:
            continue
        if "snnb::yolo_" in e.key:
            out["decode"][e.key.split("(")[0].replace("void ", "")] = {"launches": e.count, "us_per_call": total / calls}
        elif "snnb::device_input" in e.key:
            out["input_us"] += total / calls
        else:
            out["forward_us"] += total / calls
    out["decode_us"] = sum(v["us_per_call"] for v in out["decode"].values())
    return out


def detector(torch, ctx, core, modelzoo, d, args):
    from shadernn_b200._lib import check, lib
    hw, batch = (416, 416), 16
    mean4, norm4 = [127.5] * 4, [1.0 / 127.5] * 4  # the model takes [-1, 1]
    path, layers = modelzoo.build("yolov3tiny", os.path.join(d, "yolov3tiny"), input_hw=hw)
    m = core.MixedInferenceCore(ctx, path, batch=batch, input_hw=hw, fuse=True, use_cuda_graph=True)
    # BASELINE's synthetic input as 8-bit frames: few cells pass the threshold (uniform noise frames would give 100 boxes per image)
    img = np.clip(np.rint((modelzoo.synthetic_input("yolov3tiny", batch, hw) + 1.0) * 127.5), 0, 255).astype(np.uint8)
    dev_in = torch.from_numpy(img.transpose(0, 3, 1, 2).copy()).cuda()
    dev = lambda: m.detect_torch(dev_in, layout="nchw", mean4=mean4, norm4=norm4)  # noqa: E731
    hp = HostPipeline(torch, m, img, mean4, norm4, False)
    rows, cnt = np.empty((100, 6), np.float32), C.c_int()

    def host_step():  # the boxes of the previous submission are ready after its wait(): read every image's list
        waited = hp.pending is not None
        hp.step()
        if waited:
            for n in range(batch):
                check(lib().snnb_model_get_boxes(m.h, n, rows.ctypes.data_as(C.POINTER(C.c_float)), 100, C.byref(cnt)), "snnb_model_get_boxes")

    for _ in range(5):
        dev()
        host_step()
    hp.drain()
    torch.cuda.synchronize()
    rounds = []
    for _ in range(args.rounds):
        r_dev = timed(dev, args.seconds, batch, torch.cuda.synchronize)
        r_host = timed(host_step, args.seconds, batch, hp.drain)
        rounds.append({"device": r_dev, "host": r_host})
    med = lambda k: float(np.median([r[k]["frames_per_s"] for r in rounds]))  # noqa: E731
    res = {
        "shape": "%dx%d batch %d" % (hw[0], hw[1], batch),
        "device_path": "detect_torch: uint8 NCHW CUDA tensor in, rows [16, 100, 6] + counts [16] as CUDA tensors out",
        "host_path": "snnb_model_submit_u8/wait: pinned uint8 NHWC in, decode finished on the host, snnb_model_get_boxes for every image",
        "device_frames_per_s_median": med("device"),
        "host_frames_per_s_median": med("host"),
        "device_over_host": med("device") / med("host"),
        "rounds": rounds,
    }
    counts = m.detect_torch(dev_in, layout="nchw", mean4=mean4, norm4=norm4)[1]
    res["synthetic_heads"] = detector_kernel_times_us(torch, dev, 50)
    res["synthetic_heads"]["boxes_per_image"] = counts.cpu().tolist()
    m.close()
    # all-pass heads: objectness and class bias +8 for every anchor, so all 2535 cells of every image pass and NMS runs deep
    for head in [l for l in layers if l["type"] == "Conv2D" and l["outputPlanes"] == 18]:
        head["_w"]["bias"][:] = 0
        head["_w"]["bias"][[4, 5, 10, 11, 16, 17]] = 8.0
    allpass = modelzoo.write_model(layers, os.path.join(d, "yolov3tiny_allpass.json"), split=True)
    m = core.MixedInferenceCore(ctx, allpass, batch=batch, input_hw=hw, fuse=True, use_cuda_graph=True)
    dev = lambda: m.detect_torch(dev_in, layout="nchw", mean4=mean4, norm4=norm4)  # noqa: E731
    counts = m.detect_torch(dev_in, layout="nchw", mean4=mean4, norm4=norm4)[1]
    res["all_pass_heads"] = detector_kernel_times_us(torch, dev, 50)
    res["all_pass_heads"]["boxes_per_image"] = counts.cpu().tolist()
    m.close()
    return res


def torch_nv12_to_rgb(torch, frames):
    """NV12 [N, H * 3 // 2, W] uint8 -> float RGB [N, 3, H, W] (BT.601 limited range)."""
    n, rows, w = frames.shape
    h = rows // 3 * 2
    y = frames[:, :h].float() - 16.0
    uv = frames[:, h:].reshape(n, h // 2, w // 2, 2).float() - 128.0
    u = uv[..., 0].repeat_interleave(2, 1).repeat_interleave(2, 2)
    v = uv[..., 1].repeat_interleave(2, 1).repeat_interleave(2, 2)
    c = 1.164 * y
    return torch.stack([c + 1.596 * v, c - 0.391 * u - 0.813 * v, c + 2.018 * u], 1).clamp_(0.0, 255.0)


def torch_nv12_to_model(torch, frames, hw, mean4, norm4):
    """The path without run_frames: NV12 [N, H * 3 // 2, W] uint8 -> float RGB (BT.601 limited range) -> bilinear resize -> normalised
    float32 NCHW."""
    import torch.nn.functional as F
    rgb = torch_nv12_to_rgb(torch, frames)
    x = F.interpolate(rgb, size=hw, mode="bilinear", align_corners=False)
    mean = torch.tensor(mean4[:3], device=x.device).view(1, 3, 1, 1)
    norm = torch.tensor(norm4[:3], device=x.device).view(1, 3, 1, 1)
    return ((x - mean) * norm).contiguous()


def frame_kernel_us(torch, fn, calls, kernel="frame_input_kernel"):
    """Device time per call (us) of `kernel` (frame_input_kernel, frame_output_kernel, frame_roi_input_kernel, ...), from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    for _ in range(5):
        fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            fn()
        torch.cuda.synchronize()
    for e in prof.key_averages():
        if "snnb::" + kernel in e.key:
            total = getattr(e, "device_time_total", None)
            total = e.cuda_time_total if total is None else total
            return {"kernel": e.key, "launches": e.count, "us_per_batch": total / calls}
    raise RuntimeError("%s did not appear in the profile" % kernel)


def frames(torch, ctx, core, modelzoo, d, args):
    H, W = 1080, 1920
    res = []
    # (model, hw, batch, mean, norm, bytes written per model pixel: ResNet-18's input is read by its stem alone, so only the 4-channel
    # feed copy is written (2 planes x 2 bytes x 4); YOLOv3-tiny's stem reads the regular planes (2 planes x 2 bytes x 8 channels))
    cases = [("yolov3tiny", (416, 416), 16, [127.5] * 4, [1.0 / 127.5] * 4, 32), ("resnet18", (224, 224), 32, [127.5] * 4, [1.0 / 127.5] * 4, 16)]
    for name, hw, batch, mean4, norm4, out_bpp in cases:
        path, _ = modelzoo.build(name, os.path.join(d, "frames_%s" % name), input_hw=hw)
        m = core.MixedInferenceCore(ctx, path, batch=batch, input_hw=hw, fuse=True, use_cuda_graph=True)
        g = torch.Generator().manual_seed(7)
        nv12 = torch.randint(16, 236, (batch, H * 3 // 2, W), dtype=torch.uint8, generator=g).cuda()
        if name == "yolov3tiny":
            fused = lambda: m.detect_frames(nv12, mean4=mean4, norm4=norm4)  # noqa: E731
            unfused = lambda: m.detect_torch(torch_nv12_to_model(torch, nv12, hw, mean4, norm4), layout="nchw")  # noqa: E731
        else:
            fused = lambda: m.run_frames(nv12, mean4=mean4, norm4=norm4, want_classes=True)  # noqa: E731
            unfused = lambda: m.run_torch(torch_nv12_to_model(torch, nv12, hw, mean4, norm4), layout="nchw", want_classes=True)  # noqa: E731
        for _ in range(5):
            fused()
            unfused()
        torch.cuda.synchronize()
        rounds = []
        for _ in range(args.rounds):
            rounds.append({"frames": timed(fused, args.seconds, batch, torch.cuda.synchronize), "torch": timed(unfused, args.seconds, batch, torch.cuda.synchronize)})
        med = lambda k: float(np.median([r[k]["frames_per_s"] for r in rounds]))  # noqa: E731
        kt = frame_kernel_us(torch, fused, 50)
        px = batch * hw[0] * hw[1]
        written = px * out_bpp
        sampled = batch * (min(4 * hw[0] * hw[1], H * W) + 2 * min(4 * hw[0] * hw[1], (H // 2) * (W // 2)))
        whole = batch * H * W * 3 // 2
        sec = kt["us_per_batch"] * 1e-6
        kt.update({"bytes_written": written, "bytes_sampled": sampled, "bytes_whole_frames": whole,
                   "bytes_per_s_sampled": (written + sampled) / sec, "bytes_per_s_whole_frames": (written + whole) / sec})
        kt["share_of_hbm_peak_sampled"] = kt["bytes_per_s_sampled"] / HBM_BYTES_PER_S
        kt["share_of_hbm_peak_whole_frames"] = kt["bytes_per_s_whole_frames"] / HBM_BYTES_PER_S
        res.append({
            "case": "%s %dx%d batch %d from %dx%d NV12" % (name, hw[0], hw[1], batch, W, H),
            "frames_path": "detect_frames" if name == "yolov3tiny" else "run_frames (+ device classes)",
            "torch_path": "torch NV12 -> RGB + F.interpolate + normalise, then %s with float32 NCHW" % ("detect_torch" if name == "yolov3tiny" else "run_torch"),
            "frames_frames_per_s_median": med("frames"),
            "torch_frames_per_s_median": med("torch"),
            "frames_over_torch": med("frames") / med("torch"),
            "rounds": rounds,
            "frame_input_kernel": kt,
        })
        m.close()
    return res


def torch_rgb_to_nv12(torch, rgb_u8_nhwc, hw):
    """The path without transform_frames: uint8 RGB [N, h, w, 3] -> float -> F.interpolate (bilinear) to hw -> BT.601 limited-range Y, U,
    V (float) -> chroma averaged over 2 x 2 -> rounded and packed as NV12 [N, H * 3 // 2, W] uint8."""
    import torch.nn.functional as F
    x = F.interpolate(rgb_u8_nhwc.permute(0, 3, 1, 2).float(), size=hw, mode="bilinear", align_corners=False)
    r, g, b = x[:, 0], x[:, 1], x[:, 2]
    y = 0.257 * r + 0.504 * g + 0.098 * b + 16.0
    c = F.avg_pool2d(x, 2)
    u = -0.148 * c[:, 0] - 0.291 * c[:, 1] + 0.439 * c[:, 2] + 128.0
    v = 0.439 * c[:, 0] - 0.368 * c[:, 1] - 0.071 * c[:, 2] + 128.0
    uv = torch.stack([u, v], -1).reshape(x.shape[0], hw[0] // 2, hw[1])
    return torch.cat([y, uv], 1).round_().clamp_(0.0, 255.0).to(torch.uint8)


def transform(torch, ctx, core, modelzoo, d, args):
    H, W = 1080, 1920
    hw, batch = (720, 720), 8
    path, _ = modelzoo.build("candy", os.path.join(d, "transform_candy"), input_hw=hw)
    m = core.MixedInferenceCore(ctx, path, batch=batch, input_hw=hw, fuse=True, use_cuda_graph=True)
    g = torch.Generator().manual_seed(7)
    nv12 = torch.randint(16, 236, (batch, H * 3 // 2, W), dtype=torch.uint8, generator=g).cuda()
    out = torch.empty_like(nv12)
    fused = lambda: m.transform_frames(nv12, out=out)  # noqa: E731
    unfused = lambda: torch_rgb_to_nv12(torch, m.run_frames(nv12, out_dtype=torch.uint8), (H, W))  # noqa: E731
    for _ in range(5):
        fused()
        unfused()
    torch.cuda.synchronize()
    rounds = []
    for _ in range(args.rounds):
        rounds.append({"transform": timed(fused, args.seconds, batch, torch.cuda.synchronize), "torch": timed(unfused, args.seconds, batch, torch.cuda.synchronize)})
    med = lambda k: float(np.median([r[k]["frames_per_s"] for r in rounds]))  # noqa: E731
    kt = frame_kernel_us(torch, fused, 50, "frame_output_kernel")
    # written: the Y plane and the interleaved UV plane; read: Candy's 3-channel output as split-fp16 (2 planes x 8 channels x 2 bytes per
    # pixel). Every output texel lies under some frame pixel's taps at this 1.5x upscale, so the whole tensor is read.
    written = batch * (H * W + H * W // 2)
    read = batch * hw[0] * hw[1] * 2 * 8 * 2
    sec = kt["us_per_batch"] * 1e-6
    kt.update({"bytes_written": written, "bytes_read": read, "bytes_per_s": (written + read) / sec})
    kt["share_of_hbm_peak"] = kt["bytes_per_s"] / HBM_BYTES_PER_S
    res = {
        "case": "candy %dx%d batch %d from %dx%d NV12 to %dx%d NV12" % (hw[0], hw[1], batch, W, H, W, H),
        "transform_path": "transform_frames (frame_input_kernel, forward pass, frame_output_kernel)",
        "torch_path": "run_frames(out_dtype=uint8), then F.interpolate + torch RGB -> NV12 (BT.601 limited range) + packing",
        "transform_frames_per_s_median": med("transform"),
        "torch_frames_per_s_median": med("torch"),
        "transform_over_torch": med("transform") / med("torch"),
        "rounds": rounds,
        "frame_output_kernel": kt,
    }
    m.close()
    return res


def torch_luma_today(torch, m, nv12, H, W):
    """The path without transform_luma: the Y plane made dense, run_torch with uint8 in and out (Y / 255 in, 255 v out), U and V
    upsampled with F.interpolate (bilinear), and the NV12 planes packed: [N, 2H * 3 // 2, 2W] uint8."""
    import torch.nn.functional as F
    n = nv12.shape[0]
    y = nv12[:, :H].contiguous().unsqueeze(-1)
    yo = m.run_torch(y, mean4=[0.0] * 4, norm4=[1.0 / 255.0] * 4, out_dtype=torch.uint8, out_scale=255.0)[..., 0]
    uv = nv12[:, H:].reshape(n, H // 2, W // 2, 2).permute(0, 3, 1, 2).float()
    uvo = F.interpolate(uv, size=(H, W), mode="bilinear", align_corners=False).round_().clamp_(0.0, 255.0).to(torch.uint8)
    return torch.cat([yo, uvo.permute(0, 2, 3, 1).reshape(n, H, 2 * W)], 1)


def luma(torch, ctx, core, modelzoo, d, args):
    H, W = 1080, 1920
    res = []
    path, _ = modelzoo.build("espcn", os.path.join(d, "luma_espcn"), input_hw=(H, W))
    for batch in (1, 4):
        m = core.MixedInferenceCore(ctx, path, batch=batch, input_hw=(H, W), fuse=True, use_cuda_graph=True)
        g = torch.Generator().manual_seed(7)
        nv12 = torch.randint(16, 236, (batch, H * 3 // 2, W), dtype=torch.uint8, generator=g).cuda()
        out = torch.empty((batch, 2 * H * 3 // 2, 2 * W), dtype=torch.uint8, device="cuda")
        fused = lambda: m.transform_luma(nv12, norm=1.0 / 255.0, out_hw=(2 * H, 2 * W), out_scale=255.0, out=out)  # noqa: E731
        unfused = lambda: torch_luma_today(torch, m, nv12, H, W)  # noqa: E731
        for _ in range(5):
            fused()
            unfused()
        torch.cuda.synchronize()
        rounds = []
        for _ in range(args.rounds):
            rounds.append({"luma": timed(fused, args.seconds, batch, torch.cuda.synchronize), "torch": timed(unfused, args.seconds, batch, torch.cuda.synchronize)})
        med = lambda k: float(np.median([r[k]["frames_per_s"] for r in rounds]))  # noqa: E731
        kin = frame_kernel_us(torch, fused, 50, "frame_input_kernel")
        kout = frame_kernel_us(torch, fused, 50, "luma_output_kernel")
        # input: the Y plane read, the 1-channel model input written as split-fp16 (2 planes x 8 channels x 2 bytes per pixel: Cp = 8).
        # output: that same 32 bytes per pixel of ESPCN's 1-channel output read (every 32-byte sector is touched for 2 useful bytes) plus
        # the source chroma, and the out Y and UV planes written.
        kin.update({"bytes_read": batch * H * W, "bytes_written": batch * H * W * 32})
        kout.update({"bytes_read": batch * (4 * H * W * 32 + H * W // 2), "bytes_written": batch * 4 * H * W * 3 // 2})
        for kt in (kin, kout):
            # one launch per call: time per launch, as the profile can miss a launch at the edge of its window
            kt["us_per_launch"] = kt["us_per_batch"] * 50 / kt["launches"]
            kt["bytes_per_s"] = (kt["bytes_read"] + kt["bytes_written"]) / (kt["us_per_launch"] * 1e-6)
            kt["share_of_hbm_peak"] = kt["bytes_per_s"] / HBM_BYTES_PER_S
        res.append({
            "case": "espcn %dx%d batch %d from %dx%d NV12 to %dx%d NV12" % (H, W, batch, W, H, 2 * W, 2 * H),
            "luma_path": "transform_luma (frame_input_kernel<luma>, forward pass, luma_output_kernel)",
            "torch_path": "Y plane .contiguous(), run_torch (uint8 in, uint8 out), F.interpolate (bilinear) of U and V, NV12 packing",
            "luma_frames_per_s_median": med("luma"),
            "torch_frames_per_s_median": med("torch"),
            "luma_over_torch": med("luma") / med("torch"),
            "rounds": rounds,
            "frame_input_kernel": kin,
            "luma_output_kernel": kout,
        })
        m.close()
    return res


def torch_segment_today(torch, m, nv12, H, W, classes):
    """The path without segment_frames: run_frames' fp32 scores (NCHW), F.interpolate (bilinear) to the frame, then the arg-max over
    the channels (or the 0.5 threshold of one channel) and .to(uint8): [N, H, W] uint8."""
    import torch.nn.functional as F
    s = m.run_frames(nv12, mean4=[0.0] * 4, norm4=[1.0 / 255.0] * 4, out_dtype=torch.float32, out_layout="nchw")
    s = F.interpolate(s, size=(H, W), mode="bilinear", align_corners=False)
    return (s[:, 0] >= 0.5).to(torch.uint8) if classes == 1 else s.argmax(1).to(torch.uint8)


def forward_only(m, f):
    """snnb_model_run_frames with no outputs: the input kernel and the forward pass that segment_frames also runs."""
    from shadernn_b200._lib import DeviceBuffer, check, lib
    check(lib().snnb_model_run_frames(m.h, C.byref(f), (DeviceBuffer * 1)(), 0, None, m._torch_stream()), "snnb_model_run_frames")


def event_us(torch, fn, calls):
    """Device time per call (us) of `calls` back-to-back calls, between two CUDA events on the current stream."""
    for _ in range(5):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(calls):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) * 1e3 / calls


def segment(torch, ctx, core, modelzoo, d, args):
    H, W, hw, batch = 1080, 1920, (256, 256), 8
    res = []
    for classes in (1, 21):
        path, _ = modelzoo.build("unet", os.path.join(d, "seg_unet%d" % classes), input_hw=hw, classes=classes)
        m = core.MixedInferenceCore(ctx, path, batch=batch, input_hw=hw, fuse=True, use_cuda_graph=True)
        g = torch.Generator().manual_seed(11)
        nv12 = torch.randint(16, 236, (batch, H * 3 // 2, W), dtype=torch.uint8, generator=g).cuda()
        out = torch.empty((batch, H, W), dtype=torch.uint8, device="cuda")
        fused = lambda: m.segment_frames(nv12, mean4=[0.0] * 4, norm4=[1.0 / 255.0] * 4, out=out)  # noqa: E731
        unfused = lambda: torch_segment_today(torch, m, nv12, H, W, classes)  # noqa: E731
        for _ in range(5):
            fused()
            unfused()
        torch.cuda.synchronize()
        rounds = []
        for _ in range(args.rounds):
            rounds.append({"segment": timed(fused, args.seconds, batch, torch.cuda.synchronize),
                           "torch": timed(unfused, args.seconds, batch, torch.cuda.synchronize)})
        med = lambda k: float(np.median([r[k]["frames_per_s"] for r in rounds]))  # noqa: E731
        # the output kernel: CUDA events around 50 segment_frames calls, less 50 calls that run the same input kernel and forward pass
        # (run_frames with no outputs); and its device time from torch.profiler
        f = m._frames("segment", nv12, "nv12", "bt601", True, [0.0] * 4, [1.0 / 255.0] * 4)
        seg_us, fwd_us = event_us(torch, fused, 50), event_us(torch, lambda: forward_only(m, f), 50)
        kt = frame_kernel_us(torch, fused, 50, "segment_output_kernel")
        kt["us_per_launch"] = kt["us_per_batch"] * 50 / kt["launches"]
        kt["events_us_segment_call"], kt["events_us_forward_only_call"] = seg_us, fwd_us
        kt["events_us_difference"] = seg_us - fwd_us
        # bytes: the label bytes written plus the model-output planes read once (hi and lo, Cp = C rounded up to 8 fp16 per pixel each)
        cp = (classes + 7) // 8 * 8
        kt["bytes_written"] = batch * H * W
        kt["bytes_read"] = batch * hw[0] * hw[1] * cp * 2 * 2
        kt["bytes_per_s"] = (kt["bytes_read"] + kt["bytes_written"]) / (kt["us_per_launch"] * 1e-6)
        kt["share_of_hbm_peak"] = kt["bytes_per_s"] / HBM_BYTES_PER_S
        res.append({
            "case": "unet %dx%d x 1 -> %d classes, batch %d, from %dx%d NV12 to %dx%d labels" % (hw[0], hw[1], classes, batch, W, H, W, H),
            "segment_path": "segment_frames (frame_input_kernel<nv12>, forward pass, segment_output_kernel)",
            "torch_path": "run_frames(out_dtype=float32, nchw), F.interpolate (bilinear), %s, .to(uint8)" % ("s >= 0.5" if classes == 1 else "argmax(1)"),
            "segment_frames_per_s_median": med("segment"),
            "torch_frames_per_s_median": med("torch"),
            "segment_over_torch": med("segment") / med("torch"),
            "rounds": rounds,
            "segment_output_kernel": kt,
        })
        m.close()
    return res


def host_regions(rows, counts, H, W, capacity):
    """What a user computes on the host without rois_from_detections: the pixel rectangles of the first `capacity` rows (frame by frame,
    row order), each clipped to the frame; empty ones skipped."""
    out = []
    for n in range(rows.shape[0]):
        r = rows[n, :max(0, min(int(counts[n]), rows.shape[1]))]
        x0, x1 = np.floor(np.clip(r[:, 2] * W, 0, W)), np.ceil(np.clip((r[:, 2] + r[:, 4]) * W, 0, W))
        y0, y1 = np.floor(np.clip(r[:, 3] * H, 0, H)), np.ceil(np.clip((r[:, 3] + r[:, 5]) * H, 0, H))
        for i in np.nonzero((x1 > x0) & (y1 > y0))[0]:
            out.append((n, int(x0[i]), int(y0[i]), int(x1[i]), int(y1[i])))
    return out[:capacity]


def rois(torch, ctx, core, modelzoo, d, args):
    import torch.nn.functional as F
    H, W = 1080, 1920
    dhw, dbatch, chw, cbatch = (416, 416), 16, (112, 112), 64
    dmean, dnorm = [127.5] * 4, [1.0 / 127.5] * 4
    mean4, norm4 = [127.5] * 4, [1.0 / 127.5] * 4
    path, layers = modelzoo.build("yolov3tiny", os.path.join(d, "rois_yolov3tiny"), input_hw=dhw)
    for head in [l for l in layers if l["type"] == "Conv2D" and l["outputPlanes"] == 18]:  # all-pass heads (see `detector`)
        head["_w"]["bias"][:] = 0
        head["_w"]["bias"][[4, 5, 10, 11, 16, 17]] = 8.0
    det = core.MixedInferenceCore(ctx, modelzoo.write_model(layers, os.path.join(d, "rois_allpass.json"), split=True), batch=dbatch, input_hw=dhw,
                                  fuse=True, use_cuda_graph=True)
    cpath, _ = modelzoo.build("resnet18", os.path.join(d, "rois_resnet18"), input_hw=chw)
    cls = core.MixedInferenceCore(ctx, cpath, batch=cbatch, input_hw=chw, fuse=True, use_cuda_graph=True)
    g = torch.Generator().manual_seed(7)
    nv12 = torch.randint(16, 236, (dbatch, H * 3 // 2, W), dtype=torch.uint8, generator=g).cuda()
    mean_t = torch.tensor(mean4[:3], device="cuda").view(1, 3, 1, 1)
    norm_t = torch.tensor(norm4[:3], device="cuda").view(1, 3, 1, 1)

    def chain():
        r, c = det.detect_frames(nv12, mean4=dmean, norm4=dnorm)
        regions, count = ctx.rois_from_detections(r, c, (H, W), cbatch)
        return cls.run_rois(nv12, regions, count, mean4=mean4, norm4=norm4, want_classes=True)

    def today():
        r, c = det.detect_frames(nv12, mean4=dmean, norm4=dnorm)
        regions = host_regions(r.cpu().numpy(), c.cpu().numpy(), H, W, cbatch)  # synchronises
        rgb = torch_nv12_to_rgb(torch, nv12)
        crops = [F.interpolate(rgb[n:n + 1, :, y0:y1, x0:x1], size=chw, mode="bilinear", align_corners=False) for n, x0, y0, x1, y1 in regions]
        crops += [torch.zeros((cbatch - len(crops), 3) + chw, device="cuda")] if len(crops) < cbatch else []
        x = ((torch.cat(crops) - mean_t) * norm_t).contiguous()
        return cls.run_torch(x, layout="nchw", want_classes=True)

    for _ in range(5):
        chain()
        today()
    torch.cuda.synchronize()
    kept = int(ctx.rois_from_detections(*det.detect_frames(nv12, mean4=dmean, norm4=dnorm), (H, W), cbatch)[1].item())
    rounds = []
    for _ in range(args.rounds):
        rounds.append({"chain": timed(chain, args.seconds, dbatch, torch.cuda.synchronize), "today": timed(today, args.seconds, dbatch, torch.cuda.synchronize)})
    med = lambda k: float(np.median([r[k]["frames_per_s"] for r in rounds]))  # noqa: E731
    res = {"chain": {
        "case": "(a) yolov3tiny all-pass heads %dx%d batch %d from %dx%d NV12 -> %d regions -> resnet18 %dx%d batch %d" % (dhw[0], dhw[1], dbatch, W, H,
                                                                                                                       kept, chw[0], chw[1], cbatch),
        "chain_path": "detect_frames -> rois_from_detections -> run_rois (+ device classes); no host synchronisation",
        "today_path": "detect_frames, rows + counts to the host, torch NV12 -> RGB, per-box crop + F.interpolate, stack + normalise, run_torch",
        "regions_per_batch": kept,
        "chain_frames_per_s_median": med("chain"),
        "today_frames_per_s_median": med("today"),
        "chain_over_today": med("chain") / med("today"),
        "rounds": rounds,
        "kernels": {k: frame_kernel_us(torch, chain, 50, k) for k in ("rois_from_detections_kernel", "frame_roi_input_kernel", "roi_clear_kernel")},
    }}
    # (b) caller-made regions: a 2 x 2 grid of 960 x 540 cells in each frame
    rw, rh = W // 2, H // 2
    grid = [(i % dbatch, i, (i // dbatch) % 2 * rw, (i // dbatch) // 2 * rh, rw, rh) for i in range(cbatch)]
    grid_t = torch.tensor(grid, dtype=torch.int32, device="cuda")
    kt = frame_kernel_us(torch, lambda: cls.run_rois(nv12, grid_t, mean4=mean4, norm4=norm4), 50, "frame_roi_input_kernel")
    px = chw[0] * chw[1]
    written = cbatch * px * 16  # ResNet-18's stem reads the 4-channel feed copy only: 2 planes x 2 bytes x 4 per pixel
    sampled = cbatch * (min(4 * px, rw * rh) + 2 * min(4 * px, (rw // 2) * (rh // 2)))
    sec = kt["us_per_batch"] * 1e-6
    kt.update({"case": "(b) %d caller-made %dx%d regions of %dx%d NV12 frames -> resnet18 %dx%d batch %d" % (cbatch, rw, rh, W, H, chw[0], chw[1], cbatch),
               "bytes_written": written, "bytes_sampled": sampled, "bytes_per_s": (written + sampled) / sec})
    kt["share_of_hbm_peak"] = kt["bytes_per_s"] / HBM_BYTES_PER_S
    res["input_kernel"] = kt
    det.close()
    cls.close()
    return res


FRAMELIST_SIZES = [(2160, 3840)] * 4 + [(1080, 1920)] * 8 + [(720, 1280)] * 4  # (H, W) of the 16 streams


def framelist(torch, ctx, core, modelzoo, d, args):
    import torch.nn.functional as F
    dhw, chw, cbatch = (416, 416), (112, 112), 64
    dbatch = len(FRAMELIST_SIZES)
    dmean, dnorm = [127.5] * 4, [1.0 / 127.5] * 4
    mean4, norm4 = [127.5] * 4, [1.0 / 127.5] * 4
    path, layers = modelzoo.build("yolov3tiny", os.path.join(d, "list_yolov3tiny"), input_hw=dhw)
    for head in [l for l in layers if l["type"] == "Conv2D" and l["outputPlanes"] == 18]:  # all-pass heads (see `detector`)
        head["_w"]["bias"][:] = 0
        head["_w"]["bias"][[4, 5, 10, 11, 16, 17]] = 8.0
    det = core.MixedInferenceCore(ctx, modelzoo.write_model(layers, os.path.join(d, "list_allpass.json"), split=True), batch=dbatch, input_hw=dhw,
                                  fuse=True, use_cuda_graph=True)
    cpath, _ = modelzoo.build("resnet18", os.path.join(d, "list_resnet18"), input_hw=chw)
    cls = core.MixedInferenceCore(ctx, cpath, batch=cbatch, input_hw=chw, fuse=True, use_cuda_graph=True)
    g = torch.Generator().manual_seed(7)
    frames = [torch.randint(16, 236, (h * 3 // 2, w), dtype=torch.uint8, generator=g).cuda() for h, w in FRAMELIST_SIZES]  # one allocation each
    mean_t = torch.tensor(mean4[:3], device="cuda").view(1, 3, 1, 1)
    norm_t = torch.tensor(norm4[:3], device="cuda").view(1, 3, 1, 1)

    def chain():
        r, c = det.detect_frame_list(frames, mean4=dmean, norm4=dnorm)
        regions, count = ctx.rois_from_detections(r, c, FRAMELIST_SIZES, cbatch)
        return cls.run_rois_list(frames, regions, count, mean4=mean4, norm4=norm4, want_classes=True)

    def today():
        rgb = [torch_nv12_to_rgb(torch, f[None]) for f in frames]
        x = torch.cat([F.interpolate(t, size=dhw, mode="bilinear", align_corners=False) for t in rgb])
        r, c = det.detect_torch(((x - mean_t) * norm_t).contiguous(), layout="nchw")
        hr, hc = r.cpu().numpy(), c.cpu().numpy()  # synchronises
        regions = []
        for n, (h, w) in enumerate(FRAMELIST_SIZES):
            regions += [(n,) + reg[1:] for reg in host_regions(hr[n:n + 1], hc[n:n + 1], h, w, cbatch)]
        crops = [F.interpolate(rgb[n][:, :, y0:y1, x0:x1], size=chw, mode="bilinear", align_corners=False) for n, x0, y0, x1, y1 in regions[:cbatch]]
        crops += [torch.zeros((cbatch - len(crops), 3) + chw, device="cuda")] if len(crops) < cbatch else []
        return cls.run_torch(((torch.cat(crops) - mean_t) * norm_t).contiguous(), layout="nchw", want_classes=True)

    runs, med = alternate(torch, {"chain": chain, "today": today}, args.seconds, dbatch, args.rounds)
    kept = int(ctx.rois_from_detections(*det.detect_frame_list(frames, mean4=dmean, norm4=dnorm), FRAMELIST_SIZES, cbatch)[1].item())
    mix = "4 x 3840x2160 + 8 x 1920x1080 + 4 x 1280x720 NV12, each its own allocation"
    res = {"chain": {
        "case": "yolov3tiny all-pass heads %dx%d batch %d from %s -> %d regions -> resnet18 %dx%d batch %d" % (dhw[0], dhw[1], dbatch, mix, kept, chw[0],
                                                                                                           chw[1], cbatch),
        "chain_path": "detect_frame_list -> rois_from_detections (per-frame sizes) -> run_rois_list (+ device classes); no host synchronisation",
        "today_path": "per frame torch NV12 -> RGB + F.interpolate into one batch, normalise, detect_torch; rows + counts to the host; per-box crop + "
                      "F.interpolate, stack + normalise, run_torch",
        "regions_per_batch": kept,
        "chain_frames_per_s_median": med["chain"],
        "today_frames_per_s_median": med["today"],
        "chain_over_today": med["chain"] / med["today"],
        "rounds": runs,
        # the list forms of the input-side kernel templates, looked up by family: the chain runs no batch form
        "kernels": {key: frame_kernel_us(torch, chain, 50, family) for key, family in (("frame_list_input_kernel", "frame_input_kernel"),
                                                                                      ("rois_from_detections_list_kernel", "rois_from_detections_kernel"),
                                                                                      ("frame_list_roi_input_kernel", "frame_roi_input_kernel"),
                                                                                      ("roi_list_clear_kernel", "roi_clear_kernel"))},
    }}
    # the cost of the per-image descriptor: the same uniform 1080p batch through frame_input_kernel's batch and list forms
    nv12 = torch.randint(16, 236, (dbatch, 1080 * 3 // 2, 1920), dtype=torch.uint8, generator=g).cuda()
    views = [nv12[n] for n in range(dbatch)]
    batch_kt = frame_kernel_us(torch, lambda: det.detect_frames(nv12, mean4=dmean, norm4=dnorm), 50, "frame_input_kernel")
    list_kt = frame_kernel_us(torch, lambda: det.detect_frame_list(views, mean4=dmean, norm4=dnorm), 50, "frame_input_kernel")
    res["uniform_1080p"] = {"case": "yolov3tiny %dx%d batch %d from 1920x1080 NV12: the input kernel alone" % (dhw[0], dhw[1], dbatch),
                            "frame_input_kernel": batch_kt, "frame_list_input_kernel": list_kt,
                            "list_over_batch_time": list_kt["us_per_batch"] / batch_kt["us_per_batch"]}
    det.close()
    cls.close()
    return res


def framelist_out(torch, ctx, core, modelzoo, d, args):
    import torch.nn.functional as F
    n = len(FRAMELIST_SIZES)
    g = torch.Generator().manual_seed(13)
    frames = [torch.randint(16, 236, (h * 3 // 2, w), dtype=torch.uint8, generator=g).cuda() for h, w in FRAMELIST_SIZES]  # one allocation each
    uniform = torch.randint(16, 236, (n, 1080 * 3 // 2, 1920), dtype=torch.uint8, generator=g).cuda()
    views = [uniform[i] for i in range(n)]
    mix = "4 x 3840x2160 + 8 x 1920x1080 + 4 x 1280x720 NV12, each its own allocation"
    res = {}

    def entry(case, list_path, today_path, fns, list_kernel, batch_kernel, list_fn, batch_fn):
        runs, med = alternate(torch, fns, args.seconds, n, args.rounds)
        return {"case": case, "list_path": list_path, "today_path": today_path, "list_frames_per_s_median": med["list"],
                "today_frames_per_s_median": med["today"], "list_over_today": med["list"] / med["today"], "rounds": runs,
                "uniform_1080p": {list_kernel: frame_kernel_us(torch, list_fn, 50, list_kernel), batch_kernel: frame_kernel_us(torch, batch_fn, 50, batch_kernel)}}

    # Candy, in place
    hw = (720, 720)
    path, _ = modelzoo.build("candy", os.path.join(d, "listout_candy"), input_hw=hw)
    m = core.MixedInferenceCore(ctx, path, batch=n, input_hw=hw, fuse=True, use_cuda_graph=True)

    def candy_today():
        rgb = m.run_frame_list(frames, out_dtype=torch.uint8)
        for i, (h, w) in enumerate(FRAMELIST_SIZES):
            frames[i].copy_(torch_rgb_to_nv12(torch, rgb[i:i + 1], (h, w))[0])

    e = entry("candy %dx%d batch %d from and to %s (in place)" % (hw[0], hw[1], n, mix), "transform_frame_list(out=frames)",
              "run_frame_list(out_dtype=uint8), then per stream F.interpolate + torch RGB -> NV12 (BT.601 limited range) + packing into the frame",
              {"list": lambda: m.transform_frame_list(frames, out=frames), "today": candy_today}, "frame_list_output_kernel", "frame_output_kernel",
              lambda: m.transform_frame_list(views, out=views), lambda: m.transform_frames(uniform, out=uniform))
    res["transform"] = e
    m.close()
    # ESPCN, in place
    hw = (540, 960)
    path, _ = modelzoo.build("espcn", os.path.join(d, "listout_espcn"), input_hw=hw)
    m = core.MixedInferenceCore(ctx, path, batch=n, input_hw=hw, fuse=True, use_cuda_graph=True)
    kw = dict(norm=1.0 / 255.0, out_scale=255.0)

    def luma_today():
        y = torch.cat([F.interpolate(f[None, None, :h].float(), size=hw, mode="bilinear", align_corners=False) for f, (h, w) in zip(frames, FRAMELIST_SIZES)])
        yo = m.run_torch(y.round_().to(torch.uint8).permute(0, 2, 3, 1).contiguous(), mean4=[0.0] * 4, norm4=[1.0 / 255.0] * 4, out_dtype=torch.uint8,
                         out_scale=255.0)
        for i, (h, w) in enumerate(FRAMELIST_SIZES):
            up = F.interpolate(yo[i:i + 1].permute(0, 3, 1, 2).float(), size=(h, w), mode="bilinear", align_corners=False)
            frames[i][:h].copy_(up[0, 0].round_().clamp_(0.0, 255.0).to(torch.uint8))

    e = entry("espcn %dx%d batch %d from and to %s (in place)" % (hw[0], hw[1], n, mix), "transform_luma_list(out=frames)",
              "per stream F.interpolate of the Y plane to the model's size, run_torch (uint8 in, uint8 out), per stream F.interpolate back into the "
              "Y plane (chroma kept)", {"list": lambda: m.transform_luma_list(frames, out=frames, **kw), "today": luma_today}, "luma_list_output_kernel",
              "luma_output_kernel", lambda: m.transform_luma_list(views, out=views, **kw), lambda: m.transform_luma(uniform, out=uniform, **kw))
    res["luma"] = e
    m.close()
    # U-Net, 21 classes, labels at each stream's size
    hw, classes = (256, 256), 21
    path, _ = modelzoo.build("unet", os.path.join(d, "listout_unet"), input_hw=hw, classes=classes)
    m = core.MixedInferenceCore(ctx, path, batch=n, input_hw=hw, fuse=True, use_cuda_graph=True)
    sk = dict(mean4=[0.0] * 4, norm4=[1.0 / 255.0] * 4)
    labels = [torch.empty((h, w), dtype=torch.uint8, device="cuda") for h, w in FRAMELIST_SIZES]
    ulabels = torch.empty((n, 1080, 1920), dtype=torch.uint8, device="cuda")

    def seg_today():
        s = m.run_frame_list(frames, out_dtype=torch.float32, out_layout="nchw", **sk)
        for i, (h, w) in enumerate(FRAMELIST_SIZES):
            labels[i].copy_(F.interpolate(s[i:i + 1], size=(h, w), mode="bilinear", align_corners=False).argmax(1)[0].to(torch.uint8))

    e = entry("unet %dx%d x 1 -> %d classes, batch %d, from %s to labels of each stream's size" % (hw[0], hw[1], classes, n, mix), "segment_frame_list",
              "run_frame_list(out_dtype=float32, nchw), then per stream F.interpolate (bilinear) + argmax(1) + .to(uint8)",
              {"list": lambda: m.segment_frame_list(frames, out=labels, **sk), "today": seg_today}, "segment_list_output_kernel", "segment_output_kernel",
              lambda: m.segment_frame_list(views, out=[ulabels[i] for i in range(n)], **sk), lambda: m.segment_frames(uniform, out=ulabels, **sk))
    res["segment"] = e
    m.close()
    return res


def p010_surface(torch, batch, H, W, seed):
    """Random 10-bit frames as P010 words [N, H * 3 // 2, W] uint16 on the device (limited-range values, low 6 bits zero)."""
    rng = np.random.default_rng(seed)
    return torch.from_numpy((rng.integers(64, 941, (batch, H * 3 // 2, W)).astype(np.uint16) << 6)).cuda()


def torch_p010_to_nv12(torch, p010):
    """Today's workaround for 10-bit frames: every word's top 8 bits, as NV12 uint8 (one pass over the frame; the low 2 bits are lost)."""
    return ((p010.view(torch.int16) >> 8) & 0xFF).to(torch.uint8)


def alternate(torch, fns, seconds, batch, rounds):
    """Rounds of timed(fn) for each named fn, alternating, and the median frames/s of each."""
    for _ in range(5):
        for fn in fns.values():
            fn()
    torch.cuda.synchronize()
    runs = [{k: timed(fn, seconds, batch, torch.cuda.synchronize) for k, fn in fns.items()} for _ in range(rounds)]
    return runs, {k: float(np.median([r[k]["frames_per_s"] for r in runs])) for k in fns}


def with_rate(kt, read, written):
    kt["us_per_launch"] = kt["us_per_batch"] * 50 / kt["launches"]
    kt.update({"bytes_read": read, "bytes_written": written, "bytes_per_s": (read + written) / (kt["us_per_launch"] * 1e-6)})
    kt["share_of_hbm_peak"] = kt["bytes_per_s"] / HBM_BYTES_PER_S
    return kt


def p010(torch, ctx, core, modelzoo, d, args):
    """10-bit frames against 8-bit NV12 on the same sizes: detect_frames (YOLOv3-tiny 416 x 16), transform_luma (ESPCN) and
    transform_frames (Candy 720 x 8), 1920 x 1080 frames."""
    H, W = 1080, 1920
    res = []
    # YOLOv3-tiny: P010 in, against the workaround of repacking the top 8 bits as NV12
    hw, batch, mean4, norm4 = (416, 416), 16, [127.5] * 4, [1.0 / 127.5] * 4
    path, _ = modelzoo.build("yolov3tiny", os.path.join(d, "p010_yolo"), input_hw=hw)
    m = core.MixedInferenceCore(ctx, path, batch=batch, input_hw=hw, fuse=True, use_cuda_graph=True)
    src = p010_surface(torch, batch, H, W, 7)
    nv12 = torch_p010_to_nv12(torch, src)
    fns = {"p010": lambda: m.detect_frames(src, format="p010", mean4=mean4, norm4=norm4),
           "torch_repack_nv12": lambda: m.detect_frames(torch_p010_to_nv12(torch, src), mean4=mean4, norm4=norm4)}
    runs, med = alternate(torch, fns, args.seconds, batch, args.rounds)
    sampled = lambda bps: batch * (min(4 * hw[0] * hw[1], H * W) * bps + min(4 * hw[0] * hw[1], (H // 2) * (W // 2)) * 2 * bps)  # noqa: E731
    written = batch * hw[0] * hw[1] * 32
    k10 = with_rate(frame_kernel_us(torch, fns["p010"], 50), sampled(2), written)
    k8 = with_rate(frame_kernel_us(torch, lambda: m.detect_frames(nv12, mean4=mean4, norm4=norm4), 50), sampled(1), written)
    res.append({"case": "yolov3tiny 416x416 batch 16 from 1920x1080 P010", "p010_frames_per_s_median": med["p010"],
                "torch_repack_frames_per_s_median": med["torch_repack_nv12"], "p010_over_torch_repack": med["p010"] / med["torch_repack_nv12"],
                "rounds": runs, "frame_input_kernel_p010": k10, "frame_input_kernel_nv12": k8})
    m.close()
    # ESPCN: P010 -> P010 against NV12 -> NV12, 2x up
    path, _ = modelzoo.build("espcn", os.path.join(d, "p010_espcn"), input_hw=(H, W))
    m = core.MixedInferenceCore(ctx, path, batch=1, input_hw=(H, W), fuse=True, use_cuda_graph=True)
    src = p010_surface(torch, 1, H, W, 8)
    nv12 = torch_p010_to_nv12(torch, src)
    out10 = torch.empty((1, 2 * H * 3 // 2, 2 * W), dtype=torch.uint16, device="cuda")
    out8 = torch.empty((1, 2 * H * 3 // 2, 2 * W), dtype=torch.uint8, device="cuda")
    kw = dict(norm=1.0 / 255.0, out_hw=(2 * H, 2 * W), out_scale=255.0)
    fns = {"p010": lambda: m.transform_luma(src, format="p010", out=out10, **kw), "nv12": lambda: m.transform_luma(nv12, out=out8, **kw)}
    runs, med = alternate(torch, fns, args.seconds, 1, args.rounds)
    entry = {"case": "espcn 1080x1920 batch 1, 1920x1080 to 3840x2160, P010 -> P010 against NV12 -> NV12",
             "p010_frames_per_s_median": med["p010"], "nv12_frames_per_s_median": med["nv12"], "p010_over_nv12": med["p010"] / med["nv12"], "rounds": runs}
    for fmt, bps in (("p010", 2), ("nv12", 1)):
        entry["frame_input_kernel_" + fmt] = with_rate(frame_kernel_us(torch, fns[fmt], 50), H * W * bps, H * W * 32)
        entry["luma_output_kernel_" + fmt] = with_rate(frame_kernel_us(torch, fns[fmt], 50, "luma_output_kernel"),
                                                       4 * H * W * 32 + H * W // 2 * bps, 4 * H * W * 3 // 2 * bps)
    res.append(entry)
    m.close()
    # Candy: P010 -> P010 against NV12 -> NV12, 720x720 x 8, 1080p in and out
    hw, batch = (720, 720), 8
    path, _ = modelzoo.build("candy", os.path.join(d, "p010_candy"), input_hw=hw)
    m = core.MixedInferenceCore(ctx, path, batch=batch, input_hw=hw, fuse=True, use_cuda_graph=True)
    src = p010_surface(torch, batch, H, W, 9)
    nv12 = torch_p010_to_nv12(torch, src)
    out10, out8 = torch.empty_like(src), torch.empty_like(nv12)
    fns = {"p010": lambda: m.transform_frames(src, format="p010", out=out10), "nv12": lambda: m.transform_frames(nv12, out=out8)}
    runs, med = alternate(torch, fns, args.seconds, batch, args.rounds)
    entry = {"case": "candy 720x720 batch 8, 1920x1080 P010 -> 1920x1080 P010 against NV12 -> NV12",
             "p010_frames_per_s_median": med["p010"], "nv12_frames_per_s_median": med["nv12"], "p010_over_nv12": med["p010"] / med["nv12"], "rounds": runs}
    for fmt, bps in (("p010", 2), ("nv12", 1)):
        entry["frame_input_kernel_" + fmt] = with_rate(frame_kernel_us(torch, fns[fmt], 50),
                                                       batch * (H * W + H * W // 2) * bps, batch * hw[0] * hw[1] * 32)
        entry["frame_output_kernel_" + fmt] = with_rate(frame_kernel_us(torch, fns[fmt], 50, "frame_output_kernel"),
                                                        batch * hw[0] * hw[1] * 2 * 8 * 2, batch * (H * W + H * W // 2) * bps)
    res.append(entry)
    m.close()
    return res


def partial(torch, ctx, core, modelzoo, d, args):
    """Partial batches: a model loaded at its largest batch and switched with set_batch(n), against a model loaded at n and against
    padding every call to the loaded batch. Frames/s count the n useful frames of each call."""
    res = {}
    # (a) ResNet-18 224x224 run_torch, loaded at 32
    hw, big_b, mean4, norm4 = (224, 224), 32, [127.5] * 4, [1.0 / 127.5] * 4
    path, _ = modelzoo.build("resnet18", os.path.join(d, "partial_resnet18"), input_hw=hw)
    opts = dict(input_hw=hw, fuse=True, use_cuda_graph=True)
    switched = core.MixedInferenceCore(ctx, path, batch=big_b, **opts)
    padded = core.MixedInferenceCore(ctx, path, batch=big_b, **opts)
    g = torch.Generator().manual_seed(17)
    x = torch.randint(0, 256, (big_b,) + hw + (3,), dtype=torch.uint8, generator=g).cuda()
    rows = []
    for n in (1, 2, 4, 8, 16, 32):
        switched.set_batch(n)
        loaded = core.MixedInferenceCore(ctx, path, batch=n, **opts)
        xn = x[:n].contiguous()
        fns = {"set_batch": lambda: switched.run_torch(xn, mean4=mean4, norm4=norm4, want_classes=True),
               "loaded_at_n": lambda: loaded.run_torch(xn, mean4=mean4, norm4=norm4, want_classes=True),
               "padded_to_32": lambda: padded.run_torch(x, mean4=mean4, norm4=norm4, want_classes=True)}
        runs, med = alternate(torch, fns, args.seconds, n, args.rounds)
        rows.append({"n": n, "set_batch_frames_per_s_median": med["set_batch"], "loaded_at_n_frames_per_s_median": med["loaded_at_n"],
                     "padded_frames_per_s_median": med["padded_to_32"], "set_batch_over_loaded_at_n": med["set_batch"] / med["loaded_at_n"],
                     "set_batch_over_padded": med["set_batch"] / med["padded_to_32"], "rounds": runs})
        loaded.close()
    res["resnet18"] = {"case": "resnet18 224x224 loaded at batch 32, run_torch with uint8 NHWC in, float32 out and device classes; frames/s of the "
                               "n images a call needs (padded_to_32: a batch of 32 of which n are used)", "batches": rows}
    switched.close()
    padded.close()
    # (b) the framelist chain when only k of the 16 streams have a frame
    dhw, chw, cbatch = (416, 416), (112, 112), 64
    dbatch = len(FRAMELIST_SIZES)
    ypath, layers = modelzoo.build("yolov3tiny", os.path.join(d, "partial_yolov3tiny"), input_hw=dhw)
    for head in [l for l in layers if l["type"] == "Conv2D" and l["outputPlanes"] == 18]:  # all-pass heads (see `detector`)
        head["_w"]["bias"][:] = 0
        head["_w"]["bias"][[4, 5, 10, 11, 16, 17]] = 8.0
    ypath = modelzoo.write_model(layers, os.path.join(d, "partial_allpass.json"), split=True)
    det = core.MixedInferenceCore(ctx, ypath, batch=dbatch, input_hw=dhw, fuse=True, use_cuda_graph=True)
    det_pad = core.MixedInferenceCore(ctx, ypath, batch=dbatch, input_hw=dhw, fuse=True, use_cuda_graph=True)
    cpath, _ = modelzoo.build("resnet18", os.path.join(d, "partial_cls"), input_hw=chw)
    cls = core.MixedInferenceCore(ctx, cpath, batch=cbatch, input_hw=chw, fuse=True, use_cuda_graph=True)
    frames = [torch.randint(16, 236, (h * 3 // 2, w), dtype=torch.uint8, generator=g).cuda() for h, w in FRAMELIST_SIZES]
    rows = []
    for k in (4, 8, 12, 16):
        det.set_batch(k)
        # the k streams with a frame: every size class (2160p, 1080p, 720p) in the mix's proportions
        pick = [i for j in range(dbatch // 4) for i in (j, 4 + 2 * j, 5 + 2 * j, 12 + j)][:k]
        fk, sk = [frames[i] for i in pick], [FRAMELIST_SIZES[i] for i in pick]
        fpad, spad = [fk[i % k] for i in range(dbatch)], [sk[i % k] for i in range(dbatch)]

        def chain(m, fl, sizes):
            r, c = m.detect_frame_list(fl, mean4=mean4, norm4=norm4)
            regions, count = ctx.rois_from_detections(r, c, sizes, cbatch)
            return cls.run_rois_list(fl, regions, count, mean4=mean4, norm4=norm4, want_classes=True)
        fns = {"set_batch": lambda: chain(det, fk, sk), "padded_to_16": lambda: chain(det_pad, fpad, spad)}
        runs, med = alternate(torch, fns, args.seconds, k, args.rounds)
        rows.append({"k": k, "streams": sk, "set_batch_frames_per_s_median": med["set_batch"], "padded_frames_per_s_median": med["padded_to_16"],
                     "set_batch_over_padded": med["set_batch"] / med["padded_to_16"], "rounds": runs})
    res["framelist"] = {"case": "detect_frame_list (yolov3tiny all-pass heads 416x416 loaded at 16) -> rois_from_detections -> resnet18 112x112 "
                                "batch 64 run_rois_list, k of the 16 streams of `framelist` with a frame; padded_to_16 repeats the k frames "
                                "to fill the list; frames/s of the k frames", "streams": rows}
    det.close()
    det_pad.close()
    cls.close()
    return res


def counted(torch, ctx, core, modelzoo, d, args):
    """Count-sized region batches: run_rois with a device-side count on a classifier with sizes declared, against the same call with none
    declared and against set_batch(bucket(k)), the size the count selects; then the framelist chain with a few boxes per frame."""
    H, W = 1080, 1920
    chw, cbatch, sizes, nframes = (112, 112), 64, [8, 16, 32], 16
    mean4, norm4 = [127.5] * 4, [1.0 / 127.5] * 4
    cpath, _ = modelzoo.build("resnet18", os.path.join(d, "counted_resnet18"), input_hw=chw)
    opts = dict(batch=cbatch, input_hw=chw, fuse=True, use_cuda_graph=True)
    declared, undeclared, ceiling = (core.MixedInferenceCore(ctx, cpath, **opts) for _ in range(3))
    declared.set_count_batches(sizes)
    g = torch.Generator().manual_seed(7)
    nv12 = torch.randint(16, 236, (nframes, H * 3 // 2, W), dtype=torch.uint8, generator=g).cuda()
    rw, rh = W // 2, H // 2
    grid = torch.tensor([(i % nframes, i, (i // nframes) % 2 * rw, (i // nframes) // 2 * rh, rw, rh) for i in range(cbatch)], dtype=torch.int32,
                        device="cuda")
    bucket = lambda k: min([s for s in sizes if s >= k] + [cbatch])  # noqa: E731  (k = 0: the smallest declared size, the least set_batch can do)
    rows = []
    for k in (0, 1, 4, 8, 16, 24, 32, 48, 64):
        cnt = torch.tensor([k], dtype=torch.int32, device="cuda")
        ceiling.set_batch(bucket(k))
        cgrid = grid[:bucket(k)].contiguous()
        fns = {"counted": lambda: declared.run_rois(nv12, grid, cnt, mean4=mean4, norm4=norm4, want_classes=True),
               "undeclared": lambda: undeclared.run_rois(nv12, grid, cnt, mean4=mean4, norm4=norm4, want_classes=True),
               "set_batch_bucket": lambda: ceiling.run_rois(nv12, cgrid, cnt, mean4=mean4, norm4=norm4, want_classes=True)}
        runs, _ = alternate(torch, fns, args.seconds, 1, args.rounds)  # batch 1: frames/s are calls/s
        med = {key: float(np.median([r[key]["frames_per_s"] for r in runs])) for key in fns}
        rows.append({"k": k, "bucket": bucket(k), "counted_calls_per_s": med["counted"], "undeclared_calls_per_s": med["undeclared"],
                     "set_batch_bucket_calls_per_s": med["set_batch_bucket"], "counted_regions_per_s": med["counted"] * k,
                     "undeclared_regions_per_s": med["undeclared"] * k, "counted_over_undeclared": med["counted"] / med["undeclared"],
                     "counted_over_set_batch_bucket": med["counted"] / med["set_batch_bucket"], "rounds": runs})
    full = rows[-1]
    # where the overhead at k = 64 goes: the same call with one IF body (sizes [64]) and with four (sizes [8, 16, 32] and 64 itself)
    cnt = torch.tensor([cbatch], dtype=torch.int32, device="cuda")
    one = core.MixedInferenceCore(ctx, cpath, **opts)
    one.set_count_batches([cbatch])
    fns = {"four_bodies": lambda: declared.run_rois(nv12, grid, cnt, mean4=mean4, norm4=norm4, want_classes=True),
           "one_body": lambda: one.run_rois(nv12, grid, cnt, mean4=mean4, norm4=norm4, want_classes=True),
           "undeclared": lambda: undeclared.run_rois(nv12, grid, cnt, mean4=mean4, norm4=norm4, want_classes=True)}
    runs, med = alternate(torch, fns, args.seconds, 1, args.rounds)
    one.close()
    res = {"overhead_at_64": {"case": "k = 64: us per call over the undeclared call, with the bodies of sizes [8, 16, 32] and of sizes [64]",
                              "four_bodies_us": 1e6 / med["four_bodies"] - 1e6 / med["undeclared"],
                              "one_body_us": 1e6 / med["one_body"] - 1e6 / med["undeclared"], "calls_per_s_median": med, "rounds": runs}}
    res["regions"] = {
        "case": "resnet18 %dx%d loaded at %d, sizes %s declared; %d caller-made %dx%d regions of %d %dx%d NV12 frames, run_rois with a device count k "
                "(+ device classes); set_batch_bucket: a third handle after set_batch(bucket(k)), the size k selects (8 for k = 0)" % (
                    chw[0], chw[1], cbatch, sizes, cbatch, rw, rh, nframes, W, H),
        "counts": rows,
        "overhead_at_64_us": 1e6 / full["counted_calls_per_s"] - 1e6 / full["undeclared_calls_per_s"]}
    # the framelist chain with planted detector heads (scores scattered around 0.35) and a min_score that keeps a few boxes per frame
    dhw, dbatch = (416, 416), len(FRAMELIST_SIZES)
    ypath, layers = modelzoo.build("yolov3tiny", os.path.join(d, "counted_yolov3tiny"), input_hw=dhw, seed=21)
    for head in [l for l in layers if l["type"] == "Conv2D" and l["outputPlanes"] == 18]:
        head["_w"]["bias"][:] = 0
        head["_w"]["bias"][[4, 5, 10, 11]] = [-1.0, 0.0, -1.0, 0.0]
    det = core.MixedInferenceCore(ctx, modelzoo.write_model(layers, os.path.join(d, "counted_planted.json"), split=True), batch=dbatch, input_hw=dhw,
                                  fuse=True, use_cuda_graph=True)
    lists = [[torch.randint(16, 236, (h * 3 // 2, w), dtype=torch.uint8, generator=g).cuda() for h, w in FRAMELIST_SIZES] for _ in range(4)]
    r, c = det.detect_frame_list(lists[0], mean4=mean4, norm4=norm4)
    scores = np.sort(np.concatenate([r[n, :int(c[n]), 1].cpu().numpy() for n in range(dbatch)]))[::-1]
    min_score = float(scores[min(3 * dbatch, len(scores)) - 1])  # about three boxes per frame on the first list
    state = {"i": 0}

    def chain(m):
        fl = lists[state["i"] % len(lists)]
        state["i"] += 1
        rr, cc = det.detect_frame_list(fl, mean4=mean4, norm4=norm4)
        regions, count = ctx.rois_from_detections(rr, cc, FRAMELIST_SIZES, cbatch, min_score=min_score)
        return m.run_rois_list(fl, regions, count, mean4=mean4, norm4=norm4, want_classes=True)
    kept = [int(ctx.rois_from_detections(*det.detect_frame_list(fl, mean4=mean4, norm4=norm4), FRAMELIST_SIZES, cbatch, min_score=min_score)[1].item())
            for fl in lists]
    runs, med = alternate(torch, {"counted": lambda: chain(declared), "undeclared": lambda: chain(undeclared)}, args.seconds, dbatch, args.rounds)
    res["framelist_chain"] = {
        "case": "detect_frame_list (yolov3tiny planted heads %dx%d batch %d, the 16 streams of `framelist`, 4 frame sets in turn) -> "
                "rois_from_detections (min_score %.4f) -> resnet18 %dx%d batch %d run_rois_list, sizes %s declared or not" % (
                    dhw[0], dhw[1], dbatch, min_score, chw[0], chw[1], cbatch, sizes),
        "regions_per_frame_set": kept, "counted_frames_per_s_median": med["counted"], "undeclared_frames_per_s_median": med["undeclared"],
        "counted_over_undeclared": med["counted"] / med["undeclared"], "rounds": runs}
    for m in (declared, undeclared, ceiling, det):
        m.close()
    return res


def yolo_heads(modelzoo, d, name, kind, hw):
    """YOLOv3-tiny with planted heads (scores scattered around 0.35) or all-pass heads (every cell passes), as in `detector`."""
    path, layers = modelzoo.build("yolov3tiny", os.path.join(d, name), input_hw=hw, **({"seed": 21} if kind == "planted" else {}))
    for head in [l for l in layers if l["type"] == "Conv2D" and l["outputPlanes"] == 18]:
        head["_w"]["bias"][:] = 0
        head["_w"]["bias"][[4, 5, 10, 11] if kind == "planted" else [4, 5, 10, 11, 16, 17]] = [-1.0, 0.0, -1.0, 0.0] if kind == "planted" else 8.0
    return modelzoo.write_model(layers, os.path.join(d, name + "_%s.json" % kind), split=True)


def tiled(torch, ctx, core, modelzoo, d, args):
    """Sliced detection on 2160p frames: detect_rois against the torch workaround and against detect_frames of the whole frames."""
    import torch.nn.functional as F
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from _region_merge import merge_region_rows  # the float32 restatement of the merge that the tests hold detect_rois to
    H, W, nframes, hw = 2160, 3840, 4, (416, 416)
    mean4, norm4 = [127.5] * 4, [1.0 / 127.5] * 4
    tiles = [core.tile_rois((H, W), (960, 960), 96, frame=f) for f in range(nframes)]
    regions = np.concatenate([np.concatenate([t, [[f, len(t), 0, 0, W, H]]]) for f, t in enumerate(tiles)]).astype(np.int32)
    batch = len(regions)
    rois = torch.from_numpy(regions).cuda()
    g = torch.Generator().manual_seed(11)
    nv12 = torch.randint(16, 236, (nframes, H * 3 // 2, W), dtype=torch.uint8, generator=g).cuda()
    mean = torch.tensor(mean4[:3], device="cuda").view(1, 3, 1, 1)
    norm = torch.tensor(norm4[:3], device="cuda").view(1, 3, 1, 1)
    res = {"case": "%d x %dx%d NV12, %d tiles of 960x960 (>= 96 px overlap) + 1 whole-frame region per frame: %d slots into yolov3tiny %dx%d "
                   "loaded at %d; frames/s of the %d frames" % (nframes, W, H, len(tiles[0]), batch, hw[0], hw[1], batch, nframes)}
    for kind in ("planted", "allpass"):
        path = yolo_heads(modelzoo, d, "tiled_yolov3tiny", kind, hw)
        m = core.MixedInferenceCore(ctx, path, batch=batch, input_hw=hw, fuse=True, use_cuda_graph=True)
        whole = core.MixedInferenceCore(ctx, path, batch=nframes, input_hw=hw, fuse=True, use_cuda_graph=True)

        def workaround():
            rgb = torch_nv12_to_rgb(torch, nv12)
            crops = [F.interpolate(rgb[f:f + 1, :, y:y + h, x:x + w], size=hw, mode="bilinear", align_corners=False) for f, _, x, y, w, h in regions]
            r, c = m.detect_torch(((torch.cat(crops) - mean) * norm).contiguous(), layout="nchw")
            return merge_region_rows(r.cpu().numpy(), c.cpu().numpy(), regions, None, [(H, W)] * nframes, 100)
        fns = {"detect_rois": lambda: m.detect_rois(nv12, rois, mean4=mean4, norm4=norm4),
               "torch_workaround": workaround,
               "detect_frames_whole": lambda: whole.detect_frames(nv12, mean4=mean4, norm4=norm4)}
        for fn in fns.values():
            fn()
        torch.cuda.synchronize()
        runs = [{k: timed(fn, args.seconds, nframes, torch.cuda.synchronize) for k, fn in fns.items()} for _ in range(args.rounds)]
        med = {k: float(np.median([r[k]["frames_per_s"] for r in runs])) for k in fns}
        counts = m.detect_rois(nv12, rois, mean4=mean4, norm4=norm4)[1].cpu().tolist()
        # the merge kernels against the whole call, device time per call from torch.profiler
        from torch.profiler import ProfilerActivity, profile
        call = fns["detect_rois"]
        for _ in range(5):
            call()
        torch.cuda.synchronize()
        calls = 50
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(calls):
                call()
            torch.cuda.synchronize()
        merge, total = {}, 0.0
        for e in prof.key_averages():
            t = getattr(e, "device_time_total", None)
            t = e.cuda_time_total if t is None else t
            if "snnb::" not in e.key or t <= 0:
                continue
            total += t / calls
            if "snnb::roi_merge_" in e.key:
                merge[e.key.split("(")[0].replace("void ", "")] = t / calls
        merge_us = sum(merge.values())
        res[kind] = {"detect_rois_frames_per_s_median": med["detect_rois"], "torch_workaround_frames_per_s_median": med["torch_workaround"],
                     "detect_frames_whole_frames_per_s_median": med["detect_frames_whole"],
                     "detect_rois_over_torch_workaround": med["detect_rois"] / med["torch_workaround"],
                     "detect_rois_over_detect_frames_whole": med["detect_rois"] / med["detect_frames_whole"], "boxes_per_frame": counts,
                     "merge_kernels_us_per_call": merge, "merge_us_per_call": merge_us, "call_kernels_us_per_call": total,
                     "merge_share_of_call": merge_us / total if total else None, "rounds": runs}
        m.close()
        whole.close()
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--out", required=True)
    ap.add_argument("--seconds", type=float, default=2.0)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--parts", default="throughput,conversions,detector,frames",
                    help="comma-separated subset of throughput, conversions, detector, frames, transform (opt-in), rois (opt-in), luma (opt-in), "
                         "segment (opt-in), p010 (opt-in), framelist (opt-in), framelist_out (opt-in), partial (opt-in), counted (opt-in), tiled (opt-in)")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("device_io_bench: no CUDA device; this measurement needs the GPU")
    from shadernn_b200 import core, modelzoo
    os.makedirs(args.out, exist_ok=True)
    d = tempfile.mkdtemp(prefix="snnb_devio_")
    ctx = core.GpuContext(0)
    result = {"card": card(), "torch_device_name": torch.cuda.get_device_name(0)}
    parts = args.parts.split(",")
    if "throughput" in parts:
        result["throughput"] = throughput(torch, ctx, core, modelzoo, d, args)
    if "conversions" in parts:
        result["conversions"] = conversions(torch, ctx, core, modelzoo, d)
    if "detector" in parts:
        result["detector"] = detector(torch, ctx, core, modelzoo, d, args)
    if "frames" in parts:
        result["frames"] = frames(torch, ctx, core, modelzoo, d, args)
    if "transform" in parts:
        result["transform"] = transform(torch, ctx, core, modelzoo, d, args)
    if "rois" in parts:
        result["rois"] = rois(torch, ctx, core, modelzoo, d, args)
    if "luma" in parts:
        result["luma"] = luma(torch, ctx, core, modelzoo, d, args)
    if "segment" in parts:
        result["segment"] = segment(torch, ctx, core, modelzoo, d, args)
    if "framelist" in parts:
        result["framelist"] = framelist(torch, ctx, core, modelzoo, d, args)
    if "framelist_out" in parts:
        result["framelist_out"] = framelist_out(torch, ctx, core, modelzoo, d, args)
    if "p010" in parts:
        result["p010"] = p010(torch, ctx, core, modelzoo, d, args)
    if "partial" in parts:
        result["partial"] = partial(torch, ctx, core, modelzoo, d, args)
    if "counted" in parts:
        result["counted"] = counted(torch, ctx, core, modelzoo, d, args)
    if "tiled" in parts:
        result["tiled"] = tiled(torch, ctx, core, modelzoo, d, args)
    text = json.dumps(result, indent=1)
    with open(os.path.join(args.out, "device_io_bench.json"), "w") as f:
        f.write(text)
    print(text)


if __name__ == "__main__":
    main()
