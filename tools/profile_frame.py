#!/usr/bin/env python3
"""Where a frame's device time goes, kernel by kernel: one workload of bench.py (its make_scene, the same scene and frame) rendered under
torch.profiler (CUDA activity) in two modes -- single stream (RENDER_SINGLE_STREAM: one batch in flight, so no kernel's duration is
inflated by a co-resident kernel of the other batch) and the default flags (up to two batches in flight: overlapping launches each
count their full duration, so the per-kernel sums can exceed the frame).  Per mode: device ms per frame of each kernel (template
arguments kept, launch arguments dropped), the frame's device time from the library's own events, and the card's name, power limit
and SM clock read through nvidia-smi before and after, in the same run.

    python tools/profile_frame.py [--workload statue] [--frames 2] [--out profile.json]
"""
import argparse
import json
import re
import subprocess
import sys
from collections import defaultdict
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from bench import WORKLOADS, make_scene  # noqa: E402


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True, timeout=30,
                         check=True).stdout
    return dict(zip(q.split(","), [s.strip() for s in out.splitlines()[0].split(",")]))


KERNEL = re.compile(r"(k_\w+(?:<[^()]*>)?)\(")


def kernel_name(key):
    """'void pb::k_shade<1, false, false, 1>(pb::DScene, ...)' -> 'k_shade<1, false, false, 1>'; other activity (memset, memcpy) as is."""
    m = KERNEL.search(key)
    return m.group(1) if m else key


def profile_mode(gpu, h, film, stream, flags, frames):
    import torch
    from torch.profiler import ProfilerActivity, profile

    rp = h.params.contents
    rp.flags = flags
    film.zero_()
    gpu.render_device(h.params, film.data_ptr(), stream=stream)  # warm-up of this mode's launch shapes
    torch.cuda.synchronize()
    frame_ms = []
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(frames):
            film.zero_()
            st = gpu.render_device(h.params, film.data_ptr(), stream=stream)
            frame_ms.append(st["ms_total"])
        torch.cuda.synchronize()
    rp.flags = 0
    per = defaultdict(float)
    calls = defaultdict(int)
    for e in prof.key_averages():
        if e.device_time_total <= 0:
            continue
        name = kernel_name(e.key)
        per[name] += e.device_time_total / 1e3 / frames
        calls[name] += e.count
    kernels = {k: {"ms_per_frame": per[k], "launches_per_frame": calls[k] / frames} for k in sorted(per, key=per.get, reverse=True)}
    return {"frame_ms": frame_ms, "kernel_sum_ms_per_frame": sum(per.values()), "kernels": kernels}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="statue", choices=sorted(WORKLOADS))
    ap.add_argument("--frames", type=int, default=2)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("profile_frame.py needs a GPU: the render path has no CPU fallback")
    from rs_pbrt_b200 import GpuScene, _abi

    h = make_scene(args.workload)
    rp = h.params.contents
    cb = list(rp.cropped_pixel_bounds)
    film = torch.zeros((cb[3] - cb[1], cb[2] - cb[0], 4), dtype=torch.float32, device="cuda")
    stream = torch.cuda.current_stream().cuda_stream
    gpu = GpuScene(h.desc, device=0)
    torch.cuda.init()
    before = gpu_info()
    modes = {"single_stream": profile_mode(gpu, h, film, stream, _abi.RENDER_SINGLE_STREAM, args.frames),
             "default": profile_mode(gpu, h, film, stream, 0, args.frames)}
    after = gpu_info()
    gpu.close()
    result = {"workload": WORKLOADS[args.workload]["desc"], "frames": args.frames, "gpu_before": before, "gpu_after": after, "modes": modes}
    text = json.dumps(result, indent=1)
    print(text, flush=True)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(text + "\n")


if __name__ == "__main__":
    main()
