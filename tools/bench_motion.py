#!/usr/bin/env python3
"""What an animated camera costs: the statue stand-in (4.3 M triangles, 1024x1024, 128 spp, path, maxdepth 5) rendered with a static
camera, with a camera that dollies 1.5 units towards it over the shutter (the statue then fills more of the frame, so its rays cost
more), and with one that moves 0.001 units (the same image as the static one: what remains is the per-sample interpolation in
k_raygen), alternating, three frames each after one warm-up frame of each.  Prints one JSON line per frame and a summary with the card's name, power limit and SM clock (nvidia-smi, read in the same
run).  Mrays/s = BVH traversals of the frame (closest-hit + any-hit) over its device time.

    python tools/bench_motion.py [--runs 3] [--out results.json]
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    from rs_pbrt_b200 import GpuScene, scenes

    legs = {}
    for name, dolly in (("static", 0.0), ("dolly", 1.5), ("dolly_1e-3", 0.001)):
        h = scenes.statue(dolly=dolly)
        legs[name] = (h, GpuScene(h.desc, motion=h.motion))
    rows = []
    info_before = gpu_info()
    for rep in range(-1, args.runs):  # rep -1: warm-up
        for name, (h, g) in legs.items():
            _, st = g.render(h.params)
            row = dict(leg=name, rep=rep, rays=st["rays"], ms=st["ms_total"], mrays_s=st["rays"] / (st["ms_total"] * 1e3))
            if rep >= 0:
                rows.append(row)
                print(json.dumps(row), flush=True)
    summary = {"gpu_before": info_before, "gpu_after": gpu_info()}
    for name in legs:
        v = [r["mrays_s"] for r in rows if r["leg"] == name]
        summary[name] = dict(mrays_s=v, min=min(v), max=max(v))
    print(json.dumps(summary), flush=True)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(json.dumps(dict(rows=rows, summary=summary), indent=1))


if __name__ == "__main__":
    main()
