"""Motion blur through the kernel emulation (tests/emu): the -m gpu motion file, and the C ABI's handling of motion descriptions."""
import ctypes as C
import os
import shutil
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

import motion_ref
from rs_pbrt_b200 import _abi, scenes

ROOT = Path(__file__).resolve().parent.parent
pytestmark = pytest.mark.skipif(shutil.which("g++") is None, reason="needs g++")


@pytest.fixture(scope="module")
def emu():
    sys.path.insert(0, str(ROOT / "tests" / "emu"))
    import build_emu

    return _abi.bind(C.CDLL(str(build_emu.build())))


def test_gpu_motion_file_passes_through_the_emulation():
    sys.path.insert(0, str(ROOT / "tests" / "emu"))
    import build_emu

    env = dict(os.environ, RS_PBRT_B200_LIB=str(build_emu.build()))
    env.pop("PYTEST_XDIST_WORKER", None)
    r = subprocess.run([sys.executable, "-m", "pytest", str(ROOT / "tests" / "test_gpu_parity_motion.py"), "-q", "-x", "-m", "gpu", "-p", "no:xdist",
                        "-p", "no:cacheprovider"], cwd=ROOT, env=env, capture_output=True, text=True, timeout=1500)
    tail = "\n".join((r.stdout + r.stderr).splitlines()[-25:])
    assert r.returncode == 0 and " passed" in tail and "failed" not in tail, tail


def _create(emu, h, md):
    handle = C.c_void_p()
    rc = emu.pbrt_gpu_scene_create_motion(h.desc, C.byref(md), 0, C.byref(handle))
    if handle:
        emu.pbrt_gpu_scene_destroy(handle)
    return rc


def test_motion_description_validation(emu):
    h = scenes.motion_cornell(xres=8, yres=8, spp=1, n_threads=1)
    good = h.motion.contents.camera.contents
    md = _abi.PbrtMotionDesc()
    md.camera = C.pointer(good)
    assert _create(emu, h, md) == 0
    for field, k, v, want in [("end", 5, float("nan"), _abi.PBRT_E_UNSUPPORTED), ("end_inv", 0, float("inf"), _abi.PBRT_E_UNSUPPORTED),
                              ("start_time", None, float("nan"), _abi.PBRT_E_UNSUPPORTED), ("end_time", None, float("-inf"), _abi.PBRT_E_UNSUPPORTED),
                              ("start", 3, 1.0e3, _abi.PBRT_E_INVALID)]:  # a start keyframe that is not the camera's camera_to_world
        at = motion_ref.animated_transform(np.array(good.start).reshape(4, 4), np.array(good.end).reshape(4, 4), good.start_time, good.end_time)
        if k is None:
            setattr(at, field, v)
        else:
            getattr(at, field)[k] = v
        md.camera = C.pointer(at)
        assert _create(emu, h, md) == want, (field, k, v)
    assert emu.pbrt_gpu_scene_create_motion(h.desc, None, 0, None) == _abi.PBRT_E_INVALID


def test_animated_instances_stay_on_the_cpu(emu):
    import test_oracle_instancing as T

    h = T.scene("fixed", [T.translate(1.5, 0, 0.5), T.translate(-1.0, 0, 0.0)], res=(8, 8), spp=1)
    d = h.desc.contents
    ats = (_abi.PbrtAnimatedTransform * d.n_instances)()
    for i in range(d.n_instances):
        for f in ("start", "end"):
            getattr(ats[i], f)[:] = list(d.instances[i].m)
            getattr(ats[i], f + "_inv")[:] = list(d.instances[i].m_inv)
    md = _abi.PbrtMotionDesc()
    md.instances = ats
    assert _create(emu, h, md) == 0  # equal keyframes: static instances
    ats[1].end[3] += 1.0
    assert _create(emu, h, md) == _abi.PBRT_E_UNSUPPORTED
    assert b"animated object instances" in emu.pbrt_gpu_last_error()


def test_motion_struct_layout_matches_the_header(tmp_path):
    """sizeof / offsetof of the new structs as a C compiler lays them out from include/pbrt_gpu.h, against the ctypes mirror."""
    src = tmp_path / "layout.c"
    fields = {"PbrtAnimatedTransform": ["start", "start_inv", "end", "end_inv", "start_time", "end_time"], "PbrtMotionDesc": ["camera", "instances"]}
    body = "".join('printf("%s %%zu\\n", sizeof(%s));' % (s, s) + "".join('printf("%s.%s %%zu\\n", offsetof(%s, %s));' % (s, f, s, f) for f in fs)
                   for s, fs in fields.items())
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "pbrt_gpu.h"\nint main(void) { %s return 0; }\n' % body)
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-I", str(ROOT / "include"), str(src), "-o", str(exe)], check=True)
    got = dict(l.split() for l in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines())
    for s, fs in fields.items():
        ct = getattr(_abi, s)
        assert int(got[s]) == C.sizeof(ct), s
        for f in fs:
            assert int(got["%s.%s" % (s, f)]) == getattr(ct, f).offset, (s, f)


def test_keyframe_inverses_are_checked(emu):
    h = scenes.motion_cornell(xres=8, yres=8, spp=1, n_threads=1)
    good = h.motion.contents.camera.contents
    start, end = np.array(good.start).reshape(4, 4), np.array(good.end).reshape(4, 4)
    md = _abi.PbrtMotionDesc()
    for si, ei in [(np.linalg.inv(end), None), (None, np.linalg.inv(end).T), (None, np.linalg.inv(start))]:
        at = motion_ref.animated_transform(start, end, 0.0, 1.0, start_inv=si, end_inv=ei)
        md.camera = C.pointer(at)
        assert _create(emu, h, md) == _abi.PBRT_E_INVALID
        assert b"inverse" in emu.pbrt_gpu_last_error()


def test_host_camera_keyframe_is_one_matrix_when_look_at_follows_the_camera():
    """The start keyframe is the camera_to_world the Camera directive captured, m and m_inv alike, even if LookAt runs again later."""
    from rs_pbrt_b200 import HostScene

    h = HostScene()
    m = h.material(_abi.MAT_MATTE, [0.5, 0.5, 0.5, 0.0])
    h.trianglemesh(np.array([0, 1, 2], np.uint32), np.array([[0, 0, 5], [1, 0, 5], [0, 1, 5]], np.float32), material=m)
    h.light_point([0, 0, 0], [1, 1, 1])
    h.look_at([0, 0, 0], [0, 0, 1], [0, 1, 0])
    h.transform_times(0.0, 1.0)
    h.camera_motion(scenes.look_at_matrix([0.5, 0, 0], [0.5, 0, 1], [0, 1, 0]))
    h.film(8, 8)
    h.camera(fov=60.0)
    h.look_at([3, 2, 1], [0, 0, 1], [0, 1, 0])  # after the camera: does not move it
    h.sampler(1)
    h.integrator(maxdepth=1)
    h.world_end(n_threads=1)
    at = h.motion.contents.camera.contents
    start = np.array(at.start, np.float64).reshape(4, 4)
    assert np.array_equal(np.array(at.start, np.float32), np.array(h.desc.contents.camera.camera_to_world, np.float32))
    assert np.abs(start @ np.array(at.start_inv, np.float64).reshape(4, 4) - np.eye(4)).max() < 1e-5
