#!/usr/bin/env python3
"""What a goniometric light costs a frame: the statue stand-in (4.3 M triangles, 1024x1024, 128 spp, path, maxdepth 5) with one more
light above it, a goniometric light with a 48x24 map or a point light at the same place, alternating, three frames each after one
warm-up frame of each.  The difference is not the map lookup alone.  A scene with an image light runs the light-level-2 kernels
(pb_interaction.cuh), and its shade plan is one launch of the general k_shade instantiation over every class, where the point-light
scene runs the specialised Lambert and plastic instantiations; with a single launch per iteration the frame also keeps one stream
instead of overlapping two batches.  Prints one JSON line per frame and a summary with the card's name, power limit and SM clock
(nvidia-smi, read in the same run).  Mrays/s = BVH traversals over device time.

    python tools/bench_image_lights.py [--runs 3] [--out results.json]
"""
import argparse
import json
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))

from bench_motion import gpu_info  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    from rs_pbrt_b200 import GpuScene, scenes

    legs = {}
    for name in ("point", "goniometric"):
        h = scenes.statue(extra_light=name)
        legs[name] = (h, GpuScene(h.desc))
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
