"""Generator of tests/golden/conv_plan_golden.json: what the engine runs for every layer of the five BASELINE workloads at their bench
sizes (bench.WORKLOADS), for fuse 0/1, conv algo auto / simt / tcgen05 and precision fp32x3 / fp16w / fp16. Per configuration it
records the kernel each layer launches (snnb_model_layer_kernel after one timed pass; the names carry the split-K / stream-K / feed
variant), the packed weight arena's size and the launches per forward pass. Needs an H100:

    python tests/golden/make_plan_golden.py [output.json]

The fixture pins the kernel plan of the whole engine: tests/test_conv_plan.py reloads every configuration and expects the same."""
import json
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from bench import WORKLOADS  # noqa: E402

CONFIGS = [(fuse, algo, precision) for fuse in (0, 1) for algo in ("auto", "simt", "tcgen05") for precision in ("fp32x3", "fp16w", "fp16")]


def config_key(fuse, algo, precision):
    return "fuse%d/%s/%s" % (fuse, algo, precision)


def record(ctx, workload, out_dir):
    """{config key: {"kernels": [per layer], "arena_bytes": int, "launches": int}} of one workload."""
    from shadernn_b200 import core, modelzoo
    key, batch, _ = WORKLOADS[workload]
    path, _ = modelzoo.build(key, out_dir)
    got = {}
    for fuse, algo, precision in CONFIGS:
        m = core.MixedInferenceCore(ctx, path, batch=batch, conv_algo=algo, fuse=bool(fuse), precision=precision)
        try:
            m.time_layers()
            got[config_key(fuse, algo, precision)] = {"kernels": [m.layer_kernel(i) for i in range(m.num_layers)], "arena_bytes": int(m.weight_arena()[1]),
                                                      "launches": int(m.launches_per_forward)}
        finally:
            m.close()
    return got


def main(out_path):
    from shadernn_b200 import core
    ctx = core.GpuContext(0)
    fixture = {}
    for workload in sorted(WORKLOADS):
        fixture[workload] = record(ctx, workload, tempfile.mkdtemp(prefix="snnb_plan_golden_"))
        print(workload, "done", flush=True)
    with open(out_path, "w") as f:
        json.dump(fixture, f, indent=0, sort_keys=True)
    print("wrote", out_path)


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(os.path.dirname(os.path.abspath(__file__)), "conv_plan_golden.json"))
