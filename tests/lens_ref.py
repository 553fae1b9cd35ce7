"""ctypes binding of tests/lens_ref/_build/liblens_ref.so -- TEST INFRASTRUCTURE ONLY.

The oracle (oracle/, compiled in unchanged) plus an independent restatement of rs_pbrt's RealisticCamera::generate_ray_differential
and a per-sample render loop that runs li only for a camera ray weight > 0 and hands the weight to the film
(tests/lens_ref/lens_ref.cpp, on top of tests/camera_ref and tests/motion_ref).  Nothing under rs_pbrt_b200/ imports this."""
import ctypes as C
import os
import subprocess
from pathlib import Path

import numpy as np

from rs_pbrt_b200 import _abi

ROOT = Path(__file__).resolve().parent.parent
SRC = ROOT / "tests" / "lens_ref" / "lens_ref.cpp"
LIB = ROOT / "tests" / "lens_ref" / "_build" / "liblens_ref.so"
_lib = None


def build():
    deps = [SRC, ROOT / "tests" / "camera_ref" / "camera_ref.cpp", ROOT / "tests" / "motion_ref" / "motion_ref.cpp", ROOT / "include" / "pbrt_gpu.h"]
    deps += list((ROOT / "oracle").glob("*.[hc]pp"))
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
    fp, vp = C.POINTER(C.c_float), C.c_void_p
    L.orc_last_error.restype = C.c_char_p
    L.orc_init.argtypes = [C.c_char_p]
    L.orc_scene_create.argtypes = [C.POINTER(_abi.PbrtSceneDesc)]
    L.orc_scene_create.restype = vp
    L.orc_scene_destroy.argtypes = [vp]
    L.orc_scene_destroy.restype = None
    L.lref_camera_rays.argtypes = [C.POINTER(_abi.PbrtCamera), C.POINTER(_abi.PbrtRealisticLens), C.POINTER(C.c_uint32), C.POINTER(_abi.PbrtAnimatedTransform),
                                   C.c_uint32, fp, fp, fp, fp]
    L.lref_render.argtypes = [vp, C.POINTER(_abi.PbrtRealisticLens), C.POINTER(C.c_uint32), C.POINTER(_abi.PbrtAnimatedTransform), C.POINTER(_abi.PbrtRenderParams),
                              C.POINTER(C.c_int32), fp, fp, fp, C.POINTER(_abi.PbrtStats)]
    if L.orc_init(str(ROOT / "data" / "sobol_tables.bin").encode()) != 0:
        raise RuntimeError(L.orc_last_error().decode())
    _lib = L
    return L


def _fp(a):
    return a.ctypes.data_as(C.POINTER(C.c_float))


def _c(x):
    return x.contents if hasattr(x, "contents") else x


def camera_rays(camera, lens, model, p_film, p_lens, time, motion=None):
    """generate_ray_differential of each camera sample before the 1/sqrt(spp) scale: a dict of float32 arrays o, d, rx_o, ry_o, rx_d,
    ry_d (n, 3) and weight (n,); the rays are zeros where the weight is 0."""
    L = load()
    pf = np.ascontiguousarray(p_film, np.float32).reshape(-1, 2)
    n = pf.shape[0]
    pl = np.ascontiguousarray(p_lens, np.float32).reshape(n, 2)
    t = np.ascontiguousarray(np.broadcast_to(np.asarray(time, np.float32), (n,)))
    res = (C.c_uint32 * 2)(*_c(model).full_resolution)
    out = np.zeros((n, 19), np.float32)
    L.lref_camera_rays(C.byref(camera), C.byref(_c(lens)), res, C.byref(motion) if motion is not None else None, n, _fp(pf), _fp(pl), _fp(t), _fp(out))
    return dict(o=out[:, 0:3], d=out[:, 3:6], weight=out[:, 6], rx_o=out[:, 7:10], ry_o=out[:, 10:13], rx_d=out[:, 13:16], ry_d=out[:, 16:19])


class LensScene:
    """The oracle's scene of `desc` seen through the realistic camera `lens` (a PbrtRealisticLens, or a pointer to one, e.g.
    HostScene.lens) with the model's full resolution, animated when `motion` (a PbrtAnimatedTransform) is given."""

    def __init__(self, desc, model, lens, motion=None):
        self.L = load()
        self.res = (C.c_uint32 * 2)(*_c(model).full_resolution)
        self.lens = _c(lens)
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
        """-> film (h, w, 4), samples (rh, rw, spp, 3) of li's L, camera ray weights (rh, rw, spp), PbrtStats dict."""
        p = _c(params)
        cb = p.cropped_pixel_bounds
        r = np.ascontiguousarray(rect if rect is not None else list(p.sample_bounds), np.int32)
        film = np.zeros((cb[3] - cb[1], cb[2] - cb[0], 4), np.float32)
        samples = np.zeros((r[3] - r[1], r[2] - r[0], p.spp, 3), np.float32)
        weights = np.zeros((r[3] - r[1], r[2] - r[0], p.spp), np.float32)
        st = _abi.PbrtStats()
        rc = self.L.lref_render(self.h, C.byref(self.lens), self.res, C.byref(self.motion) if self.motion is not None else None, C.byref(p),
                                r.ctypes.data_as(C.POINTER(C.c_int32)), _fp(film), _fp(samples), _fp(weights), C.byref(st))
        if rc != 0:
            raise RuntimeError(self.L.orc_last_error().decode())
        return film, samples, weights, st.as_dict()
