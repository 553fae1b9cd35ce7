#!/usr/bin/env python3
"""What it costs to put one scene on N devices: N x pbrt_gpu_scene_create one after the other, N x pbrt_gpu_scene_create from one host
thread per device, and one pbrt_gpu_scene_create_multi (each large array crosses PCIe once, the replicas are completed over peer
access).  Scenes: bench.py's statue (4.3 M triangles) and landscape-64 workloads, their arrays pageable as a caller hands them over.
Every timed region ends with a synchronise of every device it used; each leg is warmed up once and timed --runs times (median and
spread reported).  Host->device bytes per device (pbrt_gpu_scene_bytes) are reported per leg.  After the timing, one
pbrt_gpu_render_multi frame over each set of scenes, and the films compared.  The card names, power limits, device count and the
peer-access matrix are read in the same run.  With one device only n = 1 runs; the multi-device figures are then reported as not
measured.

    python tools/bench_scene_multi.py [--runs 5] [--out results.json]
"""
import argparse
import json
import statistics
import subprocess
import sys
import threading
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))


def gpu_info():
    q = "index,name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        return [dict(zip(q.split(","), [s.strip() for s in line.split(",")])) for line in out.splitlines() if line.strip()]
    except Exception as e:  # the numbers are still synchronised host times; the cards are then not named
        return [{"error": str(e)}]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    import numpy as np
    import torch

    import bench
    from rs_pbrt_b200 import GpuScene, create_multi, render_multi

    n_dev = torch.cuda.device_count()
    if n_dev == 0:
        raise SystemExit("no CUDA device: nothing to measure")
    peer = [[i == j or bool(torch.cuda.can_device_access_peer(i, j)) for j in range(n_dev)] for i in range(n_dev)]

    def sync(devs):
        for d in devs:
            torch.cuda.synchronize(d)

    def timed(make, devs):
        t = []
        for k in range(args.runs + 1):  # the first run is the warm-up
            sync(devs)
            t0 = time.perf_counter()
            gs = make(devs)
            sync(devs)
            dt = time.perf_counter() - t0
            if k:
                t.append(dt * 1e3)
            keep = gs
            if k < args.runs:
                for g in gs:
                    g.close()
        return t, keep

    def sequential(devs):
        return [GpuScene(h.desc, d) for d in devs]

    def threaded(devs):
        out = [None] * len(devs)
        err = []

        def one(k):
            try:
                out[k] = GpuScene(h.desc, devs[k])
            except Exception as e:  # noqa: BLE001 (reported after the join)
                err.append(e)
        th = [threading.Thread(target=one, args=(k,)) for k in range(len(devs))]
        for t in th:
            t.start()
        for t in th:
            t.join()
        if err:
            raise err[0]
        return out

    def multi(devs):
        return create_multi(h.desc, devs)

    result = {"gpus": gpu_info(), "device_count": n_dev, "peer_access": peer, "runs": args.runs, "scenes": {}}
    for name in ("statue", "landscape-64"):
        h = bench.make_scene(name)
        d = h.desc.contents
        row = {"triangles": int(d.n_tris), "bvh_nodes": int(d.n_nodes), "legs": {}}
        counts = sorted({1, n_dev})
        for n in (2, 4, 8):
            if n < n_dev:
                counts.append(n)
        for n in sorted(set(counts)):
            devs = list(range(n))
            films = {}
            for leg, make in (("scene_create_sequential", sequential), ("scene_create_threaded", threaded), ("scene_create_multi", multi)):
                t, gs = timed(make, devs)
                film, st = render_multi(gs, h.params)
                films[leg] = film
                row["legs"]["%s_n%d" % (leg, n)] = {"n_devices": n, "ms_median": statistics.median(t), "ms_min": min(t), "ms_max": max(t),
                                                    "host_bytes_per_device": [g.upload_bytes() for g in gs], "render_multi_rays": int(st["rays"])}
                for g in gs:
                    g.close()
            ref = films["scene_create_sequential"]
            for leg, f in films.items():
                row["legs"]["%s_n%d" % (leg, n)]["film_max_abs_diff_vs_sequential"] = float(np.max(np.abs(f - ref)))
                row["legs"]["%s_n%d" % (leg, n)]["film_bit_equal_to_sequential"] = bool(np.array_equal(f.view(np.uint32), ref.view(np.uint32)))
        for n in (2, 4, 8):
            if n > n_dev:
                row["legs"]["n%d" % n] = "not measured: %d device(s) on this machine" % n_dev
        result["scenes"][name] = row
        print(json.dumps({name: row}), flush=True)
        del h
    text = json.dumps(result, indent=1)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(text + "\n")
    print(text)


if __name__ == "__main__":
    main()
