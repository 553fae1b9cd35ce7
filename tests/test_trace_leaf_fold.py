"""The wide traversal's leaf phase (pb_trace.cuh, trace_rays_wide without instances) on scenes that the statue and conference tests do not
reach: leaves of up to 15 triangles, so that one warp holds more (ray, triangle) pairs than it has lanes; coincident duplicate triangles in
one leaf and in sibling leaves, where the later primitive must win a tie in t (SURVEY.md quirk Q4); and shadow rays that exactly one
triangle of a large leaf occludes.  Any leaf phase that tests triangles out of their primitive order, or against another t_max than the
reference's running one, has to reproduce the per-lane loop's decisions here.  Every render must give the oracle's samples, film and ray
counts bit for bit -- through the kernels' source on the CPU (tests/emu), and on the GPU, where the reference-layout traversal
(PB_WIDE=0) must agree as well."""
import ctypes as C
import os
import shutil
import sys
import tempfile
from pathlib import Path

import numpy as np
import pytest

from rs_pbrt_b200 import GpuScene, HostScene, _abi

ROOT = Path(__file__).resolve().parent.parent
SMEM_BYTES = 49152  # PB_TRACE_SMEM_BYTES: smaller scenes are traced out of shared memory and never reach the wide traversal


def _matte(h, rgb):
    return h.material(_abi.MAT_MATTE, [rgb[0], rgb[1], rgb[2], 0.0])


def _quad(p0, p1, p2, p3):
    return np.array([0, 1, 2, 0, 2, 3], np.uint32), np.array([p0, p1, p2, p3], np.float32)


def _finish(h, xres, yres, spp, eye, at, maxnodeprims, direct=False):
    h.look_at(eye, at, [0, 1, 0])
    h.film(xres, yres)
    h.camera(fov=40.0)
    h.sampler(spp)
    if direct:
        h.integrator_direct(maxdepth=3, strategy="all")
    else:
        h.integrator(maxdepth=4, lightsamplestrategy="power")
    h.world_end(maxnodeprims=maxnodeprims)
    return h


def displaced_sphere(n_side=40, xres=10, yres=10, spp=2, seed=5):
    """A bumpy UV sphere like the statue's (random radial displacement, vertically stretched) over a ground quad, lit by an area light;
    its BVH is built with leaves of up to 15 primitives."""
    rng = np.random.default_rng(seed)
    h = HostScene()
    body, ground, lm = _matte(h, [0.6, 0.45, 0.3]), _matte(h, [0.4, 0.4, 0.45]), _matte(h, [0.5, 0.5, 0.5])
    u = np.linspace(0.0, 1.0, n_side + 1)
    uu, vv = np.meshgrid(u, u, indexing="xy")
    theta, phi = vv * np.pi, uu * 2.0 * np.pi
    disp = rng.random(uu.shape)
    disp[:, -1] = disp[:, 0]
    r = 1.0 + 0.08 * disp * np.sin(theta) ** 2
    P = np.stack([r * np.sin(theta) * np.cos(phi), 1.6 * r * np.cos(theta) + 1.9, r * np.sin(theta) * np.sin(phi)], -1).astype(np.float32).reshape(-1, 3)
    i = np.arange(n_side, dtype=np.uint32)[None, :]
    j = np.arange(n_side, dtype=np.uint32)[:, None]
    a = j * (n_side + 1) + i
    idx = np.stack([a, a + n_side + 1, a + 1, a + 1, a + n_side + 1, a + n_side + 2], -1).astype(np.uint32).reshape(-1)
    h.trianglemesh(idx, P, material=body)
    h.trianglemesh(*_quad([-8, 0, -8], [-8, 0, 8], [8, 0, 8], [8, 0, -8]), material=ground)
    h.trianglemesh(*_quad([-1.5, 6, -2], [1.5, 6, -2], [1.5, 6, 1], [-1.5, 6, 1]), material=lm, emit=[30.0, 28.0, 25.0])
    return _finish(h, xres, yres, spp, [0.0, 3.0, -7.0], [0.0, 1.9, 0.0], 15)


def duplicates(xres=10, yres=10, spp=2, maxnodeprims=15, seed=6):
    """A tessellated wall of which every triangle comes three times in three colours: once as written, once identical (an exact tie in
    t: the later primitive must win), once with its vertices rotated (other barycentrics, t equal or an ulp apart).  With small leaves
    the copies land in sibling leaves, with large ones in one leaf.  A stretch of bumpy terrain keeps the scene off the shared-memory
    path."""
    rng = np.random.default_rng(seed)
    h = HostScene()
    mats = [_matte(h, c) for c in ([0.8, 0.1, 0.1], [0.1, 0.8, 0.1], [0.1, 0.1, 0.8])]
    n = 6
    g = np.linspace(-2.0, 2.0, n + 1)
    gx, gy = np.meshgrid(g, g + 2.5, indexing="xy")
    P = np.stack([gx, gy, 0.3 * rng.random(gx.shape)], -1).astype(np.float32).reshape(-1, 3)
    i = np.arange(n, dtype=np.uint32)[None, :]
    j = np.arange(n, dtype=np.uint32)[:, None]
    a = j * (n + 1) + i
    tri = np.stack([a, a + 1, a + n + 1, a + 1, a + n + 2, a + n + 1], -1).astype(np.uint32).reshape(-1, 3)
    for copy, m in enumerate(mats):  # three meshes: the copies' primitive numbers are apart by the mesh size
        t = np.roll(tri, 1, axis=1) if copy == 2 else tri
        h.trianglemesh(t.reshape(-1), P, material=m)
    for k, m in enumerate(mats):  # the same within one mesh: copies next to each other in primitive order
        t = np.repeat(tri + 0, 3, axis=0)
        t[2::3] = np.roll(t[2::3], 1, axis=1)
        Pk = P + np.array([5.0 * (k - 1), 0.0, 1.5], np.float32)
        h.trianglemesh(t.reshape(-1), Pk, material=m)
    m = 40
    tg = np.linspace(-9.0, 9.0, m + 1)
    tx, tz = np.meshgrid(tg, tg, indexing="xy")
    T = np.stack([tx, 0.15 * rng.random(tx.shape), tz], -1).astype(np.float32).reshape(-1, 3)
    i = np.arange(m, dtype=np.uint32)[None, :]
    j = np.arange(m, dtype=np.uint32)[:, None]
    b = j * (m + 1) + i
    h.trianglemesh(np.stack([b, b + m + 1, b + 1, b + 1, b + m + 1, b + m + 2], -1).astype(np.uint32).reshape(-1), T, material=mats[1])
    h.trianglemesh(*_quad([-2, 9, -6], [2, 9, -6], [2, 9, -2], [-2, 9, -2]), material=_matte(h, [0.5, 0.5, 0.5]), emit=[40.0, 40.0, 40.0])
    return _finish(h, xres, yres, spp, [0.5, 3.0, -9.0], [0.0, 2.5, 0.0], maxnodeprims)


def single_occluder(xres=10, yres=10, spp=2, seed=8):
    """Clusters of 15 small triangles between a small area light and the floor, each cluster a leaf of its own: the shadow rays that
    pass through a cluster are blocked by exactly one of its triangles or by none (direct lighting: every floor point sends one)."""
    rng = np.random.default_rng(seed)
    h = HostScene()
    floor, occ, lm = _matte(h, [0.7, 0.7, 0.7]), _matte(h, [0.3, 0.3, 0.3]), _matte(h, [0.5, 0.5, 0.5])
    m = 40
    tg = np.linspace(-6.0, 6.0, m + 1)
    tx, tz = np.meshgrid(tg, tg, indexing="xy")
    T = np.stack([tx, 0.05 * rng.random(tx.shape), tz], -1).astype(np.float32).reshape(-1, 3)
    i = np.arange(m, dtype=np.uint32)[None, :]
    j = np.arange(m, dtype=np.uint32)[:, None]
    b = j * (m + 1) + i
    h.trianglemesh(np.stack([b, b + m + 1, b + 1, b + 1, b + m + 1, b + m + 2], -1).astype(np.uint32).reshape(-1), T, material=floor)
    Ps = []
    for cx in np.linspace(-1.5, 1.5, 4):
        for cz in np.linspace(-1.5, 1.5, 4):
            # 15 thin slivers side by side across the cluster, each 0.1 wide: a ray from the light crosses one of them at most
            for k in range(15):
                x0 = cx - 0.75 + 0.1 * k
                y = 2.0 + 0.002 * k
                Ps += [[x0, y, cz - 0.5], [x0 + 0.1, y, cz - 0.5], [x0 + 0.05, y, cz + 0.5]]
    P = np.array(Ps, np.float32)
    h.trianglemesh(np.arange(len(P), dtype=np.uint32), P, material=occ, two_sided=True)
    h.trianglemesh(*_quad([-0.3, 6, -0.3], [0.3, 6, -0.3], [0.3, 6, 0.3], [-0.3, 6, 0.3]), material=lm, emit=[80.0, 80.0, 80.0])
    return _finish(h, xres, yres, spp, [0.0, 5.0, -6.0], [0.0, 0.5, 0.0], 15, direct=True)


CASES = {
    "sphere-leaves-15": displaced_sphere,
    "duplicates-one-leaf": lambda **k: duplicates(maxnodeprims=15, **k),
    "duplicates-sibling-leaves": lambda **k: duplicates(maxnodeprims=1, **k),
    "single-occluder": single_occluder,
}


def _scene_bytes(h):
    d = h.desc.contents
    return int(d.n_nodes) * 32 + int(d.n_tris) * 48


def _check(lib, oracle, h):
    rp = h.params.contents
    rect = list(rp.sample_bounds)
    assert _scene_bytes(h) > SMEM_BYTES  # (the wide traversal runs for scenes in global memory only)
    g = GpuScene(h.desc, 0, lib=lib)
    try:
        gs, st = g.render_samples(h.params, rect)
        film, _ = g.render(h.params, rect=rect)
    finally:
        g.close()
    film_o, os_, so = oracle.OracleScene(h.desc).render(h.params, rect=rect, n_threads=4, want_samples=True)
    assert np.array_equal(gs.view(np.uint32), os_.view(np.uint32)), float(np.abs(gs - os_).max())
    assert np.array_equal(film[..., 3], film_o[..., 3])
    assert np.allclose(film, film_o, rtol=1e-6, atol=1e-7)
    keys = ["camera_rays", "rays", "closest_rays", "shadow_rays"]
    assert {k: st[k] for k in keys} == {k: so[k] for k in keys}
    return gs, st


@pytest.fixture(scope="module")
def emu():
    if shutil.which("g++") is None:
        pytest.skip("needs g++")
    sys.path.insert(0, str(ROOT / "tests" / "emu"))
    import build_emu
    return _abi.bind(C.CDLL(str(build_emu.build())))


@pytest.mark.parametrize("case", sorted(CASES))
def test_leaf_fold_emulated(emu, oracle, case):
    _check(emu, oracle, CASES[case]())


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(CASES))
def test_leaf_fold_gpu(oracle, product_lib, case):
    """Larger frames on the GPU against the oracle, and against the reference-layout traversal (PB_WIDE=0, read once per loaded copy of
    the library: a copy of its own)."""
    big = dict(xres=48, yres=40, spp=4)
    h = CASES[case](**big)
    gs, st = _check(product_lib, oracle, h)
    tmp = Path(tempfile.mkdtemp(prefix="pbnowide"))
    copy = tmp / "lib_nowide.so"
    shutil.copy(_abi.LIB_PATH, copy)
    old = os.environ.get("PB_WIDE")
    os.environ["PB_WIDE"] = "0"
    try:
        L = _abi.bind(C.CDLL(str(copy)))
        g = GpuScene(h.desc, 0, lib=L)
        try:
            gs0, st0 = g.render_samples(h.params, list(h.params.contents.sample_bounds))
        finally:
            g.close()
    finally:
        if old is None:
            os.environ.pop("PB_WIDE")
        else:
            os.environ["PB_WIDE"] = old
        shutil.rmtree(tmp, ignore_errors=True)
    assert np.array_equal(gs.view(np.uint32), gs0.view(np.uint32))
    assert st["rays"] == st0["rays"]
