"""ctypes binding of tests/motion_ref/_build/libmotion_ref.so -- TEST INFRASTRUCTURE ONLY.

The oracle (oracle/, compiled in unchanged) plus an independent restatement of rs_pbrt's AnimatedTransform and a per-sample render
loop for an animated camera (tests/motion_ref/motion_ref.cpp).  Nothing under rs_pbrt_b200/ imports this."""
import ctypes as C
import subprocess
from pathlib import Path

import numpy as np

from rs_pbrt_b200 import _abi

ROOT = Path(__file__).resolve().parent.parent
SRC = ROOT / "tests" / "motion_ref" / "motion_ref.cpp"
LIB = ROOT / "tests" / "motion_ref" / "_build" / "libmotion_ref.so"
_lib = None


def build():
    deps = [SRC, ROOT / "include" / "pbrt_gpu.h"] + list((ROOT / "oracle").glob("*.[hc]pp"))
    if not LIB.exists() or any(s.stat().st_mtime > LIB.stat().st_mtime for s in deps):
        LIB.parent.mkdir(exist_ok=True)
        tmp = LIB.with_suffix(".so.tmp%d" % __import__("os").getpid())
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
    L.mref_interpolate.argtypes = [C.POINTER(_abi.PbrtAnimatedTransform), C.c_uint32, fp, fp, fp]
    L.mref_decompose.argtypes = [fp, fp, fp, fp]
    L.mref_decompose.restype = None
    L.mref_render.argtypes = [vp, C.POINTER(_abi.PbrtAnimatedTransform), C.POINTER(_abi.PbrtRenderParams), C.POINTER(C.c_int32), fp, fp, fp,
                              C.POINTER(_abi.PbrtStats)]
    if L.orc_init(str(ROOT / "data" / "sobol_tables.bin").encode()) != 0:
        raise RuntimeError(L.orc_last_error().decode())
    _lib = L
    return L


def _fp(a):
    return a.ctypes.data_as(C.POINTER(C.c_float))


def animated_transform(start, end, start_time=0.0, end_time=1.0, start_inv=None, end_inv=None):
    """PbrtAnimatedTransform of two 4x4 keyframes (inverses in f64 when not given)."""
    a = _abi.PbrtAnimatedTransform()
    for name, m in (("start", start), ("end", end)):
        m = np.asarray(m, np.float32).reshape(4, 4)
        inv = start_inv if name == "start" else end_inv
        inv = np.asarray(inv if inv is not None else np.linalg.inv(m.astype(np.float64)), np.float32).reshape(4, 4)
        getattr(a, name)[:] = m.reshape(-1).tolist()
        getattr(a, name + "_inv")[:] = inv.reshape(-1).tolist()
    a.start_time, a.end_time = start_time, end_time
    return a


def interpolate(at, times):
    """AnimatedTransform::interpolate at each time: (m, m_inv), each (n, 4, 4) float32."""
    L = load()
    t = np.ascontiguousarray(times, np.float32).reshape(-1)
    m = np.zeros((t.size, 16), np.float32)
    mi = np.zeros((t.size, 16), np.float32)
    L.mref_interpolate(C.byref(at), t.size, _fp(t), _fp(m), _fp(mi))
    return m.reshape(-1, 4, 4), mi.reshape(-1, 4, 4)


def decompose(m):
    """AnimatedTransform::decompose: translation (3,), quaternion (x, y, z, w), scale matrix (4, 4)."""
    L = load()
    mm = np.ascontiguousarray(m, np.float32).reshape(16)
    t, q, s = np.zeros(3, np.float32), np.zeros(4, np.float32), np.zeros(16, np.float32)
    L.mref_decompose(_fp(mm), _fp(t), _fp(q), _fp(s))
    return t, q, s.reshape(4, 4)


class MotionScene:
    """The oracle's scene of `desc`, rendered through an animated camera (`camera`: a PbrtAnimatedTransform, or None)."""

    def __init__(self, desc, camera=None):
        self.L = load()
        self.camera = camera
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
        rc = self.L.mref_render(self.h, C.byref(self.camera) if self.camera is not None else None, C.byref(p), r.ctypes.data_as(C.POINTER(C.c_int32)),
                                _fp(film), _fp(samples), _fp(times), C.byref(st))
        if rc != 0:
            raise RuntimeError(self.L.orc_last_error().decode())
        return film, samples, times, st.as_dict()
