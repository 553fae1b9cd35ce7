"""pbrt_gpu_scene_create_multi through the kernel emulation (tests/emu): the -m gpu file on three emulated devices, with and without peer
access between them, and the C ABI's refusals."""
import ctypes as C
import os
import shutil
import subprocess
import sys
from pathlib import Path

import pytest

from rs_pbrt_b200 import _abi, scenes

ROOT = Path(__file__).resolve().parent.parent
pytestmark = pytest.mark.skipif(shutil.which("g++") is None, reason="needs g++")


@pytest.fixture(scope="module")
def emu():
    sys.path.insert(0, str(ROOT / "tests" / "emu"))
    import build_emu

    return _abi.bind(C.CDLL(str(build_emu.build())))


@pytest.mark.parametrize("peer", ["peer", "no-peer"])
def test_gpu_scene_multi_file_passes_through_the_emulation(peer):
    """Device memory comes back poisoned (PB_EMU_POISON), so a slice that no device wrote cannot pass by luck."""
    sys.path.insert(0, str(ROOT / "tests" / "emu"))
    import build_emu

    env = dict(os.environ, RS_PBRT_B200_LIB=str(build_emu.build()), PB_EMU_DEVICES="3", PB_EMU_POISON="0xff")
    if peer == "no-peer":
        env["PB_EMU_NO_PEER"] = "1"
    env.pop("PYTEST_XDIST_WORKER", None)
    r = subprocess.run([sys.executable, "-m", "pytest", str(ROOT / "tests" / "test_gpu_scene_multi.py"), "-q", "-m", "gpu", "-p", "no:xdist",
                        "-p", "no:cacheprovider"], cwd=ROOT, env=env, capture_output=True, text=True, timeout=1500)
    tail = "\n".join((r.stdout + r.stderr).splitlines()[-25:])
    assert r.returncode == 0 and " passed" in tail and "failed" not in tail and "skipped" not in tail, tail


def _multi(emu, desc, devices, n=None, motion=None):
    """rc, the handles (pre-set to garbage, so that the call has to clear them) and pbrt_gpu_last_error"""
    n = len(devices) if n is None else n
    out = (C.c_void_p * max(n, 1))(*([0x1234] * max(n, 1)))
    devs = (C.c_int * max(len(devices), 1))(*devices) if devices is not None else None
    rc = emu.pbrt_gpu_scene_create_multi(desc, motion, devs, n, out)
    handles = list(out)[:n]
    if rc == 0:
        for h in handles:
            emu.pbrt_gpu_scene_destroy(h)
    return rc, handles, emu.pbrt_gpu_last_error()


def _single(emu, desc):
    out = C.c_void_p()
    rc = emu.pbrt_gpu_scene_create(desc, 0, C.byref(out))
    if out:
        emu.pbrt_gpu_scene_destroy(out)
    return rc, emu.pbrt_gpu_last_error()


def test_refusals(emu, monkeypatch):
    monkeypatch.setenv("PB_EMU_DEVICES", "3")
    h = scenes.cornell_box(xres=8, yres=8, spp=1, n_threads=1)
    assert _multi(emu, h.desc, [0, 1, 2])[0] == 0
    assert _multi(emu, None, [0, 1])[0] == _abi.PBRT_E_INVALID
    assert emu.pbrt_gpu_scene_create_multi(h.desc, None, None, 2, (C.c_void_p * 2)()) == _abi.PBRT_E_INVALID
    assert emu.pbrt_gpu_scene_create_multi(h.desc, None, (C.c_int * 2)(0, 1), 2, None) == _abi.PBRT_E_INVALID
    assert _multi(emu, h.desc, [0], n=0)[0] == _abi.PBRT_E_INVALID
    rc, out, err = _multi(emu, h.desc, [0, 1, 0])
    assert rc == _abi.PBRT_E_INVALID and b"twice" in err and not any(out)
    rc, out, _ = _multi(emu, h.desc, list(range(17)))
    assert rc == _abi.PBRT_E_UNSUPPORTED and not any(out)
    # a bad ordinal in the last place: refused before any replica is made, every handle null, and the devices stay usable
    for bad in (7, -1):
        rc, out, err = _multi(emu, h.desc, [0, 1, bad])
        assert rc == _abi.PBRT_E_INVALID and b"ordinal" in err and not any(out), bad
    assert _multi(emu, h.desc, [2, 0, 1])[0] == 0


def test_description_errors_are_those_of_scene_create(emu, monkeypatch):
    """A fault the host finds (an unknown light kind) and one the device finds while it flattens the triangles, after every replica's
    uploads and peer copies (a vertex index out of range): the same code and text as pbrt_gpu_scene_create, and no replica left."""
    monkeypatch.setenv("PB_EMU_DEVICES", "3")
    for fault in ("light", "vertex"):
        h = scenes.cornell_box(xres=8, yres=8, spp=1, n_threads=1)
        d = h.desc.contents
        if fault == "light":
            d.lights[0].kind = 99
        else:
            d.tris[d.n_tris - 1].v[1] = 1 << 30
        rc, err = _single(emu, h.desc)
        assert rc < 0
        for devs in ([0], [0, 1, 2]):
            mrc, out, merr = _multi(emu, h.desc, devs)
            assert (mrc, merr) == (rc, err) and not any(out), (fault, devs)
    h = scenes.cornell_box(xres=8, yres=8, spp=1, n_threads=1)
    assert _multi(emu, h.desc, [0, 1, 2])[0] == 0
