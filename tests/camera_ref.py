"""ctypes binding of tests/camera_ref/_build/libcamera_ref.so -- TEST INFRASTRUCTURE ONLY.

The oracle (oracle/, compiled in unchanged) plus independent restatements of rs_pbrt's OrthographicCamera and EnvironmentCamera and
a per-sample render loop that traces their rays, animated or not (tests/camera_ref/camera_ref.cpp, on top of tests/motion_ref).
Nothing under rs_pbrt_b200/ imports this."""
import ctypes as C
import os
import subprocess
from pathlib import Path

import numpy as np

from rs_pbrt_b200 import _abi

ROOT = Path(__file__).resolve().parent.parent
SRC = ROOT / "tests" / "camera_ref" / "camera_ref.cpp"
LIB = ROOT / "tests" / "camera_ref" / "_build" / "libcamera_ref.so"
_lib = None

KINDS = {"perspective": _abi.PBRT_CAMERA_PERSPECTIVE, "orthographic": _abi.PBRT_CAMERA_ORTHOGRAPHIC, "environment": _abi.PBRT_CAMERA_ENVIRONMENT}


def build():
    deps = [SRC, ROOT / "tests" / "motion_ref" / "motion_ref.cpp", ROOT / "include" / "pbrt_gpu.h"] + list((ROOT / "oracle").glob("*.[hc]pp"))
    if not LIB.exists() or any(s.stat().st_mtime > LIB.stat().st_mtime for s in deps):
        LIB.parent.mkdir(exist_ok=True)
        tmp = LIB.with_suffix(".so.tmp%d" % os.getpid())
        subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-pthread", "-shared", "-o", str(tmp), str(SRC)], check=True)
        tmp.replace(LIB)
    return LIB


def load():
    global _lib
    if _lib is not None:
        return _lib
    build()
    L = C.CDLL(str(LIB))
    fp, vp, u32p = C.POINTER(C.c_float), C.c_void_p, C.POINTER(C.c_uint32)
    L.orc_last_error.restype = C.c_char_p
    L.orc_init.argtypes = [C.c_char_p]
    L.orc_scene_create.argtypes = [C.POINTER(_abi.PbrtSceneDesc)]
    L.orc_scene_create.restype = vp
    L.orc_scene_destroy.argtypes = [vp]
    L.orc_scene_destroy.restype = None
    L.cref_camera_rays.argtypes = [C.POINTER(_abi.PbrtCamera), C.c_uint32, u32p, C.c_uint32, C.c_uint32, fp, fp, fp, fp]
    L.cref_render.argtypes = [vp, C.c_uint32, u32p, C.POINTER(_abi.PbrtAnimatedTransform), C.POINTER(_abi.PbrtRenderParams), C.POINTER(C.c_int32), fp, fp, fp,
                              C.POINTER(_abi.PbrtStats)]
    if L.orc_init(str(ROOT / "data" / "sobol_tables.bin").encode()) != 0:
        raise RuntimeError(L.orc_last_error().decode())
    _lib = L
    return L


def _fp(a):
    return a.ctypes.data_as(C.POINTER(C.c_float))


def _model(model):
    m = model.contents if hasattr(model, "contents") else model
    return int(m.kind), (C.c_uint32 * 2)(*m.full_resolution)


def camera_rays(camera, model, p_film, time, p_lens, spp=1):
    """The reference's camera rays after camera_to_world and the 1/sqrt(spp) scale: a dict of float32 arrays o, d (n, 3), time (n,),
    has_diff (n,) and rx_o, ry_o, rx_d, ry_d (n, 3)."""
    L = load()
    kind, res = _model(model)
    pf = np.ascontiguousarray(p_film, np.float32).reshape(-1, 2)
    n = pf.shape[0]
    t = np.ascontiguousarray(np.broadcast_to(np.asarray(time, np.float32), (n,)))
    pl = np.ascontiguousarray(np.broadcast_to(np.asarray(p_lens, np.float32).reshape(-1, 2), (n, 2)))
    out = np.zeros((n, 20), np.float32)
    L.cref_camera_rays(C.byref(camera), kind, res, spp, n, _fp(pf), _fp(t), _fp(pl), _fp(out))
    return dict(o=out[:, 0:3], d=out[:, 3:6], time=out[:, 6], has_diff=out[:, 7] != 0.0, rx_o=out[:, 8:11], ry_o=out[:, 11:14], rx_d=out[:, 14:17],
                ry_d=out[:, 17:20])


class CameraScene:
    """The oracle's scene of `desc`, rendered through camera `model` (a PbrtCameraModel, or a pointer to one, e.g. HostScene.camera_model),
    animated when `motion` (a PbrtAnimatedTransform) is given."""

    def __init__(self, desc, model, motion=None):
        self.L = load()
        self.kind, self.res = _model(model)
        self.motion = motion
        self.h = self.L.orc_scene_create(desc)
        if not self.h:
            raise RuntimeError(self.L.orc_last_error().decode())

    def close(self):
        if self.h:
            self.L.orc_scene_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def render(self, params, rect=None):
        """-> film (h, w, 4), samples (rh, rw, spp, 3), ray times (rh, rw, spp), PbrtStats dict."""
        p = params.contents if hasattr(params, "contents") else params
        cb = p.cropped_pixel_bounds
        r = np.ascontiguousarray(rect if rect is not None else list(p.sample_bounds), np.int32)
        film = np.zeros((cb[3] - cb[1], cb[2] - cb[0], 4), np.float32)
        samples = np.zeros((r[3] - r[1], r[2] - r[0], p.spp, 3), np.float32)
        times = np.zeros((r[3] - r[1], r[2] - r[0], p.spp), np.float32)
        st = _abi.PbrtStats()
        rc = self.L.cref_render(self.h, self.kind, self.res, C.byref(self.motion) if self.motion is not None else None, C.byref(p),
                                r.ctypes.data_as(C.POINTER(C.c_int32)), _fp(film), _fp(samples), _fp(times), C.byref(st))
        if rc != 0:
            raise RuntimeError(self.L.orc_last_error().decode())
        return film, samples, times, st.as_dict()
