"""Goniometric and projection lights through the kernel emulation (tests/emu): the -m gpu file, the C ABI's validation of the two kinds,
and PbrtLight's layout against a C compiler."""
import ctypes as C
import os
import shutil
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

from rs_pbrt_b200 import _abi, scenes

ROOT = Path(__file__).resolve().parent.parent
pytestmark = pytest.mark.skipif(shutil.which("g++") is None, reason="needs g++")


@pytest.fixture(scope="module")
def emu():
    sys.path.insert(0, str(ROOT / "tests" / "emu"))
    import build_emu

    return _abi.bind(C.CDLL(str(build_emu.build())))


def test_gpu_image_light_file_passes_through_the_emulation():
    sys.path.insert(0, str(ROOT / "tests" / "emu"))
    import build_emu

    env = dict(os.environ, RS_PBRT_B200_LIB=str(build_emu.build()))
    env.pop("PYTEST_XDIST_WORKER", None)
    r = subprocess.run([sys.executable, "-m", "pytest", str(ROOT / "tests" / "test_gpu_image_lights.py"), "-q", "-m", "gpu", "-p", "no:xdist",
                        "-p", "no:cacheprovider"], cwd=ROOT, env=env, capture_output=True, text=True, timeout=1500)
    tail = "\n".join((r.stdout + r.stderr).splitlines()[-25:])
    assert r.returncode == 0 and " passed" in tail and "failed" not in tail, tail


def _create(emu, h):
    handle = C.c_void_p()
    rc = emu.pbrt_gpu_scene_create(h.desc, 0, C.byref(handle))
    if rc == 0:
        emu.pbrt_gpu_scene_destroy(handle)
    return rc


def _image_light(h):
    d = h.desc.contents
    return next(d.lights[i] for i in range(d.n_lights) if d.lights[i].kind in (_abi.LIGHT_GONIOMETRIC, _abi.LIGHT_PROJECTION))


@pytest.mark.parametrize("kind", ["goniometric", "projection"])
def test_valid_scene_is_accepted(emu, kind):
    assert _create(emu, scenes.cornell_box(xres=4, yres=4, spp=1, lights=kind)) == 0


@pytest.mark.parametrize("kind", ["goniometric", "projection"])
@pytest.mark.parametrize("field,value,status", [
    ("env_res", (0, 24), -1),
    ("env_res", (16385, 1), -2),
    ("p", (float("nan"), 0.0, 0.0), -1),
    ("p", (0.0, float("inf"), 0.0), -1),
    ("w2l", (float("nan"),) + (0.0,) * 8, -1),
])
def test_invalid_light_is_rejected(emu, kind, field, value, status):
    h = scenes.cornell_box(xres=4, yres=4, spp=1, lights=kind)
    arr = getattr(_image_light(h), field)
    for k, v in enumerate(value):
        arr[k] = v
    assert _create(emu, h) == status


@pytest.mark.parametrize("fov", [0.0, -10.0, 180.0, float("nan"), float("inf")])
def test_projection_fov_out_of_range_is_rejected(emu, fov):
    h = scenes.cornell_box(xres=4, yres=4, spp=1, lights="projection")
    _image_light(h).fov = fov
    assert _create(emu, h) == -1


def test_projection_without_map_is_rejected(emu):
    h = scenes.cornell_box(xres=4, yres=4, spp=1, lights="projection")
    _image_light(h).env_texels = None
    assert _create(emu, h) == -1


def test_point_light_read_as_goniometric_renders(emu):
    """a point light record whose kind says goniometric is a goniometric light without a map: it renders"""
    h = scenes.cornell_box(xres=4, yres=4, spp=1, lights="point")
    d = h.desc.contents
    d.lights[0].kind = _abi.LIGHT_GONIOMETRIC
    handle = C.c_void_p()
    assert emu.pbrt_gpu_scene_create(h.desc, 0, C.byref(handle)) == 0
    rp = h.params.contents
    film = np.zeros((4, 4, 4), np.float32)
    rect = (C.c_int32 * 4)(*list(rp.sample_bounds))
    assert emu.pbrt_gpu_render(handle, h.params, rect, film.ctypes.data_as(C.POINTER(C.c_float)), C.byref(_abi.PbrtStats())) == 0
    emu.pbrt_gpu_scene_destroy(handle)
    assert np.all(np.isfinite(film)) and film[..., :3].sum() > 0


def test_pbrt_light_layout_matches_c(tmp_path):
    src = tmp_path / "layout.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "pbrt_gpu.h"\nint main(void) { printf("%zu %zu %zu %d %d\\n", sizeof(PbrtLight), '
                   'offsetof(PbrtLight, fov), offsetof(PbrtLight, n_samples), PBRT_LIGHT_GONIOMETRIC, PBRT_LIGHT_PROJECTION); return 0; }\n')
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-std=c99", "-I", str(ROOT / "include"), str(src), "-o", str(exe)], check=True)
    size, off_fov, off_ns, kg, kp = map(int, subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split())
    assert (size, off_fov, off_ns) == (C.sizeof(_abi.PbrtLight), _abi.PbrtLight.fov.offset, _abi.PbrtLight.n_samples.offset)
    assert off_fov == off_ns + 4 and (kg, kp) == (_abi.LIGHT_GONIOMETRIC, _abi.LIGHT_PROJECTION)
