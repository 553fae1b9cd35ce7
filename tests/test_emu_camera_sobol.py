"""k_raygen's camera samples come from per-render Sobol' tables (k_camera_sobol: index = F[s] ^ X[x] ^ Y[y]).  The kernels' source
on the CPU (tests/emu) against the oracle, bit for bit per sample, at the edges of that split: a 1x1 frame (resolution exponent m = 0,
every index 0) through each integrator that draws camera samples, and a path-integrator frame whose batches split the pixel's samples
(first_sample > 0) on a frame width that is not a power of two."""
import ctypes as C
import os
import shutil
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

from rs_pbrt_b200 import GpuScene, _abi, scenes

ROOT = Path(__file__).resolve().parent.parent
pytestmark = pytest.mark.skipif(shutil.which("g++") is None, reason="needs g++")


@pytest.fixture(scope="module")
def emu():
    sys.path.insert(0, str(ROOT / "tests" / "emu"))
    import build_emu
    return _abi.bind(C.CDLL(str(build_emu.build())))


@pytest.mark.parametrize("integrator", ["path", ("direct", "all"), "whitted", ("ao", 4, True)])
def test_one_pixel_frame(emu, oracle, integrator):
    h = scenes.cornell_box(xres=1, yres=1, spp=8, integrator=integrator, materials="mixed")
    rp = h.params.contents
    sb = list(rp.sample_bounds)
    assert (sb[2] - sb[0], sb[3] - sb[1]) == (1, 1)  # resolution 1: m = 0
    g = GpuScene(h.desc, 0, lib=emu)
    try:
        gs, st = g.render_samples(h.params, sb)
        film, _ = g.render(h.params, rect=sb)
    finally:
        g.close()
    film_o, so, sto = oracle.OracleScene(h.desc).render(h.params, rect=sb, n_threads=4, want_samples=True)
    assert np.array_equal(gs.view(np.uint32), so.view(np.uint32)), float(np.abs(gs - so).max())
    assert np.array_equal(film[..., 3], film_o[..., 3])
    assert np.allclose(film, film_o, rtol=1e-6, atol=1e-7)
    assert st["camera_rays"] == sto["camera_rays"] == 8 and st["rays"] == sto["rays"]


def test_path_batches_split_the_pixel_samples(emu, tmp_path):
    """PB_BATCH_LOG2 = 10 (read once per process, hence the subprocess) against 2048 spp: every batch holds 1024 samples of one pixel, half
    of them starting at sample 1024."""
    script = tmp_path / "run.py"
    script.write_text('''
import sys, ctypes as C, numpy as np
sys.path.insert(0, %r); sys.path.insert(0, %r)
from rs_pbrt_b200 import GpuScene, _abi, scenes
import oracle_lib
emu = _abi.bind(C.CDLL(%r))
h = scenes.cornell_box(xres=3, yres=2, spp=2048, maxdepth=2)
sb = list(h.params.contents.sample_bounds)
g = GpuScene(h.desc, 0, lib=emu)
gs, st = g.render_samples(h.params, sb)
fo, so, sto = oracle_lib.OracleScene(h.desc).render(h.params, rect=sb, n_threads=4, want_samples=True)
assert np.array_equal(gs.view(np.uint32), so.view(np.uint32)), float(np.abs(gs - so).max())
assert st["camera_rays"] == sto["camera_rays"] and st["rays"] == sto["rays"], (st, sto)
assert st["trace_launches"] >= 12 * 3, st["trace_launches"]  # 6 pixels x 2 sample halves, one batch each
print("ok")
''' % (str(ROOT), str(ROOT / "tests"), str(ROOT / "tests" / "emu" / "_build" / "librs_pbrt_b200_emu.so")))
    env = dict(os.environ, PB_BATCH_LOG2="10")
    r = subprocess.run([sys.executable, str(script)], env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), r.stdout[-2000:] + r.stderr[-2000:]
