"""The realistic camera through the kernel emulation (tests/emu): the -m gpu realistic-camera file, the C ABI's refusals of lenses,
the layout of the new structs, and the other cameras unchanged by the new entry point."""
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


def test_gpu_realistic_file_passes_through_the_emulation():
    sys.path.insert(0, str(ROOT / "tests" / "emu"))
    import build_emu

    env = dict(os.environ, RS_PBRT_B200_LIB=str(build_emu.build()))
    env.pop("PYTEST_XDIST_WORKER", None)
    r = subprocess.run([sys.executable, "-m", "pytest", str(ROOT / "tests" / "test_gpu_parity_realistic.py"), "-q", "-x", "-m", "gpu", "-p", "no:xdist",
                        "-p", "no:cacheprovider"], cwd=ROOT, env=env, capture_output=True, text=True, timeout=2400)
    tail = "\n".join((r.stdout + r.stderr).splitlines()[-25:])
    assert r.returncode == 0 and " passed" in tail and "failed" not in tail, tail


def _create(emu, desc, model, lens, devices=(0,)):
    devs = (C.c_int * max(len(devices), 1))(*devices)
    out = (C.c_void_p * max(len(devices), 1))()
    rc = emu.pbrt_gpu_scene_create_lens(desc, None, C.byref(model) if model is not None else None, C.byref(lens) if lens is not None else None, devs,
                                        len(devices), out)
    for h in out:
        if h:
            emu.pbrt_gpu_scene_destroy(h)
    return rc, list(out)


@pytest.fixture(scope="module")
def lens_scene():
    return scenes.cornell_box(xres=8, yres=6, spp=1, n_threads=1, camera="realistic")


def _copy_lens(h):
    src = h.lens.contents
    el = (_abi.PbrtLensElement * (_abi.PBRT_MAX_LENS_ELEMENTS + 1))()
    for i in range(src.n_elements):
        el[i] = src.elements[i]
    b = (C.c_float * 256)(*[src.exit_pupil_bounds[i] for i in range(256)])
    lens = _abi.PbrtRealisticLens(C.cast(el, C.POINTER(_abi.PbrtLensElement)), src.n_elements, C.cast(b, C.POINTER(C.c_float)), src.film_diagonal,
                                  src.simple_weighting)
    return lens, el, b


def test_lens_validation(emu, lens_scene):
    h = lens_scene
    M = _abi.PbrtCameraModel
    model = M(_abi.PBRT_CAMERA_REALISTIC, (8, 6))
    lens, el, b = _copy_lens(h)
    assert _create(emu, h.desc, model, lens)[0] == 0
    for kind in (_abi.PBRT_CAMERA_PERSPECTIVE, _abi.PBRT_CAMERA_ORTHOGRAPHIC, _abi.PBRT_CAMERA_ENVIRONMENT, 7):
        rc, out = _create(emu, h.desc, M(kind, (8, 6)), lens)
        assert rc == _abi.PBRT_E_INVALID and not any(out), kind
    assert _create(emu, h.desc, None, lens)[0] == _abi.PBRT_E_INVALID
    # lens == NULL is pbrt_gpu_scene_create_camera: the realistic kind needs its lens
    rc, _ = _create(emu, h.desc, model, None)
    assert rc == _abi.PBRT_E_UNSUPPORTED and b"camera kind" in emu.pbrt_gpu_last_error()
    for res in ((0, 6), (8, 0)):
        assert _create(emu, h.desc, M(_abi.PBRT_CAMERA_REALISTIC, res), lens)[0] == _abi.PBRT_E_INVALID
    n = lens.n_elements

    def bad(mutate, code=_abi.PBRT_E_INVALID):
        lens2, el2, b2 = _copy_lens(h)
        mutate(lens2, el2, b2)
        rc, out = _create(emu, h.desc, model, lens2)
        assert rc == code and not any(out), rc

    bad(lambda l, e, q: setattr(l, "n_elements", 0))
    bad(lambda l, e, q: setattr(l, "n_elements", _abi.PBRT_MAX_LENS_ELEMENTS + 1), _abi.PBRT_E_UNSUPPORTED)
    bad(lambda l, e, q: setattr(l, "film_diagonal", 0.0))
    bad(lambda l, e, q: setattr(l, "film_diagonal", float("nan")))
    bad(lambda l, e, q: setattr(e[n - 1], "thickness", float("inf")))
    bad(lambda l, e, q: setattr(e[0], "eta", float("nan")))
    bad(lambda l, e, q: q.__setitem__(4 * 10, q[4 * 10 + 2] + 1.0))  # pmin.x > pmax.x
    bad(lambda l, e, q: q.__setitem__(4 * 63 + 3, float("nan")))
    bad(lambda l, e, q: setattr(l, "elements", None))
    bad(lambda l, e, q: setattr(l, "exit_pupil_bounds", None))
    lens2, el2, b2 = _copy_lens(h)
    lens2.n_elements = _abi.PBRT_MAX_LENS_ELEMENTS  # the limit itself is accepted
    for i in range(n, _abi.PBRT_MAX_LENS_ELEMENTS):
        el2[i] = _abi.PbrtLensElement(0.0, 0.0, 0.0, 1.0)
    assert _create(emu, h.desc, model, lens2)[0] == 0


def test_structs_layout_matches_the_header(tmp_path):
    """sizeof / offsetof of PbrtLensElement and PbrtRealisticLens, PBRT_CAMERA_REALISTIC and PBRT_MAX_LENS_ELEMENTS as a C compiler sees
    include/pbrt_gpu.h, against the ctypes mirror; PbrtCameraModel keeps its 12 bytes."""
    src = tmp_path / "layout.c"
    fields = [("PbrtLensElement", f) for f, _ in _abi.PbrtLensElement._fields_] + [("PbrtRealisticLens", f) for f, _ in _abi.PbrtRealisticLens._fields_]
    body = "".join('printf("%s.%s %%zu\\n", offsetof(%s, %s));\n' % (s, f, s, f) for s, f in fields)
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "pbrt_gpu.h"\nint main(void) {\n' + body +
                   'printf("elem %zu\\nlens %zu\\nmodel %zu\\n", sizeof(PbrtLensElement), sizeof(PbrtRealisticLens), sizeof(PbrtCameraModel));\n'
                   'printf("kind %d\\nmax %d\\n", PBRT_CAMERA_REALISTIC, PBRT_MAX_LENS_ELEMENTS); return 0; }\n')
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-I", str(ROOT / "include"), str(src), "-o", str(exe)], check=True)
    got = dict(l.split() for l in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines())
    for s, f in fields:
        assert int(got["%s.%s" % (s, f)]) == getattr(getattr(_abi, s), f).offset, (s, f)
    assert int(got["elem"]) == C.sizeof(_abi.PbrtLensElement) == 16
    assert int(got["lens"]) == C.sizeof(_abi.PbrtRealisticLens)
    assert int(got["model"]) == C.sizeof(_abi.PbrtCameraModel) == 12
    assert (int(got["kind"]), int(got["max"])) == (_abi.PBRT_CAMERA_REALISTIC, _abi.PBRT_MAX_LENS_ELEMENTS)


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


@pytest.mark.parametrize("camera,kw", [("perspective", dict(textures="ewa")), ("perspective", dict(integrator=("direct", "all"))),
                                       ("orthographic", dict(textures="trilinear")), ("environment", dict(integrator="whitted", materials="mixed"))],
                         ids=["persp-ewa", "persp-direct", "ortho-trilinear", "env-whitted"])
def test_other_cameras_render_like_create_camera(emu, camera, kw):
    """pbrt_gpu_scene_create_lens with lens == NULL (camera NULL or a model) gives pbrt_gpu_scene_create_camera's samples."""
    h = scenes.cornell_box(xres=10, yres=8, spp=4, n_threads=1, camera=camera, **kw)
    models = [h.camera_model] + ([None] if camera == "perspective" else [])
    for model in models:
        a = (C.c_void_p * 1)()
        assert emu.pbrt_gpu_scene_create_camera(h.desc, None, model, (C.c_int * 1)(0), 1, a) == 0
        base = _samples(emu, h, a[0])
        b = (C.c_void_p * 1)()
        assert emu.pbrt_gpu_scene_create_lens(h.desc, None, model, None, (C.c_int * 1)(0), 1, b) == 0
        got = _samples(emu, h, b[0])
        assert np.array_equal(got[0].view(np.uint32), base[0].view(np.uint32)) and got[1] == base[1]


def test_host_mirror_lens_units_and_aperture_clamp():
    """RealisticCamera::new's units (mm -> m, diameter -> radius) and the stop's aperture: replaced by aperturediameter unless that is
    larger than the file's; the last thickness is the focused one."""
    h = scenes.cornell_box(xres=8, yres=6, spp=1, n_threads=1, camera="realistic", aperturediameter=8.0)
    L = h.lens.contents
    rows = np.array(scenes.DGAUSS_50MM, np.float32)
    el = np.array([[L.elements[i].curvature_radius, L.elements[i].thickness, L.elements[i].eta, L.elements[i].aperture_radius] for i in range(L.n_elements)],
                  np.float32)
    assert L.n_elements == len(rows) and abs(L.film_diagonal - 0.035) < 1e-9
    assert np.array_equal(el[:, 0], rows[:, 0] * np.float32(0.001)) and np.array_equal(el[:-1, 1], rows[:-1, 1] * np.float32(0.001))
    stop = int(np.argmax(rows[:, 0] == 0))
    assert el[stop, 3] == np.float32(8.0) * np.float32(0.001) / np.float32(2.0)
    others = np.arange(len(rows)) != stop
    assert np.array_equal(el[others, 3], rows[others, 3] * np.float32(0.001) / np.float32(2.0))
    assert 0.030 < el[-1, 1] < 0.045  # a 50 mm double-Gauss focused at 1000 units: the back focal distance
    h2 = scenes.cornell_box(xres=8, yres=6, spp=1, n_threads=1, camera="realistic", aperturediameter=40.0)  # larger than the stop: clamped
    assert h2.lens.contents.elements[stop].aperture_radius == np.float32(17.1) * np.float32(0.001) / np.float32(2.0)
