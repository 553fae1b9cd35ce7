#!/usr/bin/env python3
"""What the realistic camera costs: the statue stand-in (4.3 M triangles, 1024x1024, 128 spp, path, maxdepth 5) through the
perspective camera and through the realistic camera (scenes.DGAUSS_50MM on a 35 mm film, focused on the statue), from the same eye,
alternating, three frames each after one warm-up frame of each.  Per frame: Mrays/s (BVH traversals over device time), the samples
the lens vignettes (1 - camera_rays / samples).  Then, in a run of its own under torch.profiler, the device time of k_raygen per frame
for each camera: the realistic camera's ray generation traces up to five rays through the lens per sample, and the difference over the
perspective k_raygen, per camera sample, is the cost of that lens trace.  The card's name, power limit and SM clock come from
nvidia-smi in the same run.

    python tools/bench_realistic.py [--runs 3] [--out results.json]
"""
import argparse
import json
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        return dict(zip(q.split(","), [s.strip() for s in out.splitlines()[0].split(",")]))
    except Exception as e:  # the numbers are still device-timed; the card is then not named
        return {"error": str(e)}


def raygen_ms(g, h, frames):
    """Device time of the k_raygen launches of `frames` frames (torch.profiler, CUDA activity), per frame."""
    import torch
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(frames):
            g.render(h.params)
        torch.cuda.synchronize()
    us = sum(e.device_time_total for e in prof.key_averages() if "k_raygen" in e.key)
    return us / 1e3 / frames


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    from rs_pbrt_b200 import GpuScene, scenes

    legs = {}
    for kind in ("perspective", "realistic"):
        h = scenes.statue(camera=kind)
        legs[kind] = (h, GpuScene(h.desc, camera=h.camera_model, lens=h.lens))
    samples = 1024 * 1024 * 128
    rows = []
    info_before = gpu_info()
    for rep in range(-1, args.runs):  # rep -1: warm-up
        for name, (h, g) in legs.items():
            _, st = g.render(h.params)
            row = dict(leg=name, rep=rep, rays=st["rays"], camera_rays=st["camera_rays"], ms=st["ms_total"], mrays_s=st["rays"] / (st["ms_total"] * 1e3),
                       vignetted_fraction=1.0 - st["camera_rays"] / samples)
            if rep >= 0:
                rows.append(row)
                print(json.dumps(row), flush=True)
    prof = {name: raygen_ms(g, h, 2) for name, (h, g) in legs.items()}
    summary = {"gpu_before": info_before, "gpu_after": gpu_info(), "samples_per_frame": samples, "k_raygen_ms_per_frame": prof,
               "lens_trace_ns_per_sample": (prof["realistic"] - prof["perspective"]) * 1e6 / samples}
    for name in legs:
        v = [r["mrays_s"] for r in rows if r["leg"] == name]
        summary[name] = dict(mrays_s=v, min=min(v), max=max(v), vignetted_fraction=[r for r in rows if r["leg"] == name][-1]["vignetted_fraction"])
    print(json.dumps(summary), flush=True)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(json.dumps(dict(rows=rows, summary=summary), indent=1))


if __name__ == "__main__":
    main()
