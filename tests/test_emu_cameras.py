"""Orthographic and environment cameras through the kernel emulation (tests/emu): the -m gpu camera file, the C ABI's refusals of
camera models, and the layout of the new struct."""
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


def test_gpu_camera_file_passes_through_the_emulation():
    sys.path.insert(0, str(ROOT / "tests" / "emu"))
    import build_emu

    env = dict(os.environ, RS_PBRT_B200_LIB=str(build_emu.build()))
    env.pop("PYTEST_XDIST_WORKER", None)
    r = subprocess.run([sys.executable, "-m", "pytest", str(ROOT / "tests" / "test_gpu_parity_cameras.py"), "-q", "-x", "-m", "gpu", "-p", "no:xdist",
                        "-p", "no:cacheprovider"], cwd=ROOT, env=env, capture_output=True, text=True, timeout=2400)
    tail = "\n".join((r.stdout + r.stderr).splitlines()[-25:])
    assert r.returncode == 0 and " passed" in tail and "failed" not in tail, tail


def _create(emu, desc, model, devices=(0,), motion=None):
    devs = (C.c_int * max(len(devices), 1))(*devices)
    out = (C.c_void_p * max(len(devices), 1))()
    rc = emu.pbrt_gpu_scene_create_camera(desc, motion, C.byref(model) if model is not None else None, devs, len(devices), out)
    for h in out:
        if h:
            emu.pbrt_gpu_scene_destroy(h)
    return rc, [h for h in out]


def test_camera_model_validation(emu):
    h = scenes.cornell_box(xres=8, yres=6, spp=1, n_threads=1)
    M = _abi.PbrtCameraModel
    for kind in (_abi.PBRT_CAMERA_PERSPECTIVE, _abi.PBRT_CAMERA_ORTHOGRAPHIC, _abi.PBRT_CAMERA_ENVIRONMENT):
        assert _create(emu, h.desc, M(kind, (8, 6)))[0] == 0, kind
    assert _create(emu, h.desc, None)[0] == 0
    for kind in (3, 7, 0xFFFFFFFF):  # 3: RealisticCamera, outside the GPU path like any kind this version does not know
        rc, out = _create(emu, h.desc, M(kind, (8, 6)))
        assert rc == _abi.PBRT_E_UNSUPPORTED and not any(out), kind
        assert b"camera kind" in emu.pbrt_gpu_last_error()
    for res in ((0, 6), (8, 0), (0, 0)):
        rc, out = _create(emu, h.desc, M(_abi.PBRT_CAMERA_ENVIRONMENT, res))
        assert rc == _abi.PBRT_E_INVALID and not any(out), res
        assert b"full_resolution" in emu.pbrt_gpu_last_error()
    # the other kinds do not read full_resolution
    assert _create(emu, h.desc, M(_abi.PBRT_CAMERA_ORTHOGRAPHIC, (0, 0)))[0] == 0
    assert _create(emu, h.desc, M(_abi.PBRT_CAMERA_ENVIRONMENT, (8, 6)), devices=())[0] == _abi.PBRT_E_INVALID
    assert _create(emu, h.desc, M(_abi.PBRT_CAMERA_ENVIRONMENT, (8, 6)), devices=(0, 0))[0] == _abi.PBRT_E_INVALID
    out = (C.c_void_p * 1)()
    assert emu.pbrt_gpu_scene_create_camera(None, None, None, (C.c_int * 1)(0), 1, out) == _abi.PBRT_E_INVALID
    assert emu.pbrt_gpu_scene_create_camera(h.desc, None, None, None, 1, out) == _abi.PBRT_E_INVALID
    assert emu.pbrt_gpu_scene_create_camera(h.desc, None, None, (C.c_int * 1)(0), 1, None) == _abi.PBRT_E_INVALID


def test_a_bad_description_fails_alike_with_any_camera(emu):
    """A description error is reported with the same code and text whatever the camera model."""
    h = scenes.cornell_box(xres=8, yres=6, spp=1, n_threads=1)
    d = h.desc.contents
    saved = d.tris[3].material
    d.tris[3].material = d.n_materials + 5
    try:
        out = C.c_void_p()
        rc0 = emu.pbrt_gpu_scene_create(h.desc, 0, C.byref(out))
        e0 = emu.pbrt_gpu_last_error()
        for kind in (_abi.PBRT_CAMERA_ORTHOGRAPHIC, _abi.PBRT_CAMERA_ENVIRONMENT):
            rc, out2 = _create(emu, h.desc, _abi.PbrtCameraModel(kind, (8, 6)))
            assert (rc, emu.pbrt_gpu_last_error()) == (rc0, e0) and rc0 == _abi.PBRT_E_INVALID and not any(out2)
    finally:
        d.tris[3].material = saved


def test_camera_model_layout_matches_the_header(tmp_path):
    """sizeof / offsetof of PbrtCameraModel and the kind values as a C compiler sees include/pbrt_gpu.h, against the ctypes mirror."""
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "pbrt_gpu.h"\nint main(void) {\n'
                   'printf("size %zu\\n", sizeof(PbrtCameraModel)); printf("kind %zu\\n", offsetof(PbrtCameraModel, kind));\n'
                   'printf("full_resolution %zu\\n", offsetof(PbrtCameraModel, full_resolution));\n'
                   'printf("persp %d\\northo %d\\nenv %d\\n", PBRT_CAMERA_PERSPECTIVE, PBRT_CAMERA_ORTHOGRAPHIC, PBRT_CAMERA_ENVIRONMENT);\n'
                   'printf("camera %zu\\nscene %zu\\n", sizeof(PbrtCamera), sizeof(PbrtSceneDesc)); return 0; }\n')
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-I", str(ROOT / "include"), str(src), "-o", str(exe)], check=True)
    got = dict(l.split() for l in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines())
    M = _abi.PbrtCameraModel
    assert int(got["size"]) == C.sizeof(M) == 12
    assert int(got["kind"]) == M.kind.offset and int(got["full_resolution"]) == M.full_resolution.offset
    assert (int(got["persp"]), int(got["ortho"]), int(got["env"])) == (_abi.PBRT_CAMERA_PERSPECTIVE, _abi.PBRT_CAMERA_ORTHOGRAPHIC, _abi.PBRT_CAMERA_ENVIRONMENT)
    # the existing structs keep their sizes
    assert int(got["camera"]) == C.sizeof(_abi.PbrtCamera) == 144 and int(got["scene"]) == C.sizeof(_abi.PbrtSceneDesc)


def test_abi_version_is_unchanged(emu):
    assert emu.pbrt_gpu_abi_version() == 4


def _samples(emu, h, handle):
    rect = np.ascontiguousarray(list(h.params.contents.sample_bounds), np.int32)
    n = int((rect[2] - rect[0]) * (rect[3] - rect[1]) * h.params.contents.spp)
    buf = np.zeros(3 * n, np.float32)
    st = _abi.PbrtStats()
    rc = emu.pbrt_gpu_render_samples(handle, h.params, rect.ctypes.data_as(C.POINTER(C.c_int32)), buf.ctypes.data_as(C.POINTER(C.c_float)), C.byref(st))
    emu.pbrt_gpu_scene_destroy(handle)
    assert rc == 0, emu.pbrt_gpu_last_error()
    return buf, (st.camera_rays, st.rays, st.closest_rays, st.shadow_rays)


@pytest.mark.parametrize("kw", [dict(textures="ewa"), dict(integrator=("direct", "all"), textures="trilinear"), dict(lensradius=20.0, focaldistance=800.0)],
                         ids=["ewa", "direct-trilinear", "lens"])
def test_null_and_perspective_models_render_like_scene_create(emu, kw):
    h = scenes.cornell_box(xres=10, yres=8, spp=4, n_threads=1, **kw)
    plain = C.c_void_p()
    assert emu.pbrt_gpu_scene_create(h.desc, 0, C.byref(plain)) == 0
    base = _samples(emu, h, plain)
    for model in (None, C.byref(_abi.PbrtCameraModel(_abi.PBRT_CAMERA_PERSPECTIVE, (10, 8)))):
        out = (C.c_void_p * 1)()
        assert emu.pbrt_gpu_scene_create_camera(h.desc, None, model, (C.c_int * 1)(0), 1, out) == 0
        got = _samples(emu, h, out[0])
        assert np.array_equal(got[0].view(np.uint32), base[0].view(np.uint32)) and got[1] == base[1]


def test_host_mirror_camera_model():
    """HostScene hands the kind and the full film resolution (not the crop window's) to the library; the orthographic raster_to_camera
    maps the raster corners onto the screen window."""
    h = scenes.cornell_box(xres=16, yres=10, spp=1, n_threads=1, camera="environment", crop=[0.25, 0.75, 0.0, 0.5])
    m = h.camera_model.contents
    assert (m.kind, tuple(m.full_resolution)) == (_abi.PBRT_CAMERA_ENVIRONMENT, (16, 10))
    sw = [-3.0, 5.0, -1.0, 2.0]
    h = scenes.cornell_box(xres=16, yres=10, spp=1, n_threads=1, camera="orthographic", screenwindow=sw)
    m = h.camera_model.contents
    assert (m.kind, tuple(m.full_resolution)) == (_abi.PBRT_CAMERA_ORTHOGRAPHIC, (16, 10))
    r2c = np.array(h.desc.contents.camera.raster_to_camera, np.float64).reshape(4, 4)
    for raster, cam in [((0, 0), (-3.0, 2.0)), ((16, 10), (5.0, -1.0)), ((8, 5), (1.0, 0.5))]:
        q = r2c @ np.array([raster[0], raster[1], 0.0, 1.0])
        np.testing.assert_allclose(q[:3] / q[3], [cam[0], cam[1], 0.0], atol=1e-5)
    h = scenes.cornell_box(xres=16, yres=10, spp=1, n_threads=1)
    assert h.camera_model.contents.kind == _abi.PBRT_CAMERA_PERSPECTIVE


@pytest.mark.parametrize("kind,kw", [("orthographic", dict(lensradius=30.0, focaldistance=850.0, shutter=(0.1, 0.9))), ("orthographic", dict()),
                                     ("environment", dict(shutter=(0.25, 0.5)))], ids=["ortho-lens-shutter", "ortho", "environment"])
def test_export_writes_the_camera_and_reads_back(tmp_path, kind, kw):
    """pbrt_export writes the Camera directive of each kind (screen window, lens, shutter); tests/pbrt_reader_cameras.py reads it back
    to the same camera, the same model and the same reference render."""
    import camera_ref
    import pbrt_reader_cameras
    from rs_pbrt_b200 import pbrt_export

    h = scenes.cornell_box(xres=12, yres=10, spp=2, n_threads=1, camera=kind, **kw)
    pbrt_export.write(h, tmp_path / "scene.pbrt")
    text = (tmp_path / "scene.pbrt").read_text()
    assert ('Camera "%s"' % kind) in text
    h2 = pbrt_reader_cameras.read(tmp_path / "scene.pbrt", n_threads=1)
    c1, c2 = h.desc.contents.camera, h2.desc.contents.camera
    for f in ("raster_to_camera", "camera_to_world"):
        assert np.array_equal(np.array(getattr(c1, f)), np.array(getattr(c2, f))), f
    assert (c1.lens_radius, c1.focal_distance, c1.shutter_open, c1.shutter_close) == (c2.lens_radius, c2.focal_distance, c2.shutter_open, c2.shutter_close)
    m1, m2 = h.camera_model.contents, h2.camera_model.contents
    assert (m1.kind, tuple(m1.full_resolution)) == (m2.kind, tuple(m2.full_resolution))
    _, s1, _, st1 = camera_ref.CameraScene(h.desc, m1).render(h.params)
    _, s2, _, st2 = camera_ref.CameraScene(h2.desc, m2).render(h2.params)
    assert np.array_equal(s1, s2) and st1["rays"] == st2["rays"]
