"""pbrt_gpu_scene_create_multi on hardware: every replica renders like a scene pbrt_gpu_scene_create made on the same device -- every
sample bit for bit, every work counter --, render_multi over the replicas gives the film it gives over separately created scenes, a
replica outlives its siblings, and each large array crosses PCIe once in all.  Also run on the CPU through the kernel emulation with
three emulated devices, with and without peer access (test_emu_scene_multi.py)."""
import os

import numpy as np
import pytest

from rs_pbrt_b200 import GpuScene, _abi, create_multi, render_multi, scenes

pytestmark = pytest.mark.gpu
EMULATED = bool(os.environ.get("RS_PBRT_B200_LIB"))


def device_count():
    if EMULATED:
        return int(os.environ.get("PB_EMU_DEVICES", "1"))
    import torch

    return torch.cuda.device_count()


def peer_everywhere(n):
    if EMULATED:
        return not int(os.environ.get("PB_EMU_NO_PEER", "0"))
    import torch

    return all(torch.cuda.can_device_access_peer(i, j) for i in range(n) for j in range(n) if i != j)


N_ALL = device_count()
STATUE_SIDE = 40 if EMULATED else 160  # 160: 51 200 triangles, past the shared-memory traversal, so the wide records are built too

SCENES = {
    "cornell-mixed": lambda: scenes.cornell_box(xres=10, yres=8, spp=4, materials="mixed", lights="delta", n_threads=1),
    "statue": lambda: scenes.statue(n_side=STATUE_SIDE, xres=8, yres=8, spp=2),
    "landscape-fixed": lambda: scenes.landscape(xres=10, yres=6, spp=2, n_trees=20, grid=8, detail=6, instancing="fixed"),
    "landscape-reference": lambda: scenes.landscape(xres=10, yres=6, spp=2, n_trees=20, grid=8, detail=6, instancing="reference"),
    "textures": lambda: scenes.cornell_box(xres=8, yres=8, spp=2, textures="ewa+float+graph+bump", n_threads=1),
    "infinite": lambda: scenes.sky_scene(xres=8, yres=8, spp=2, env="two"),
    "goniometric": lambda: scenes.cornell_box(xres=8, yres=8, spp=2, lights="goniometric", n_threads=1),
    "projection": lambda: scenes.cornell_box(xres=8, yres=8, spp=2, lights="projection", n_threads=1),
    "alpha": lambda: scenes.cornell_box(xres=8, yres=8, spp=2, alpha="masks", n_threads=1),
    "motion": lambda: scenes.motion_cornell(xres=8, yres=8, spp=2, pan=12.0, n_threads=1),
}
# all devices first: the replicas are made before a single scene of the same description could leave its buffers in a device's cache
CASES = [(name, n) for name in SCENES for n in sorted({N_ALL, 1}, reverse=True)]


def samples_and_counters(g, h):
    rp = h.params.contents
    old = rp.flags
    rp.flags = old | _abi.RENDER_COUNT_WORK
    try:
        got, st = g.render_samples(h.params, list(rp.sample_bounds))
    finally:
        rp.flags = old
    return got, {k: v for k, v in st.items() if not k.startswith("ms_")}


@pytest.mark.parametrize("name,n", CASES, ids=["%s-n%d" % c for c in CASES])
def test_replicas_render_like_single_scenes(name, n):
    h = SCENES[name]()
    reps = create_multi(h.desc, list(range(n)), motion=h.motion)
    got = [samples_and_counters(g, h) for g in reps]
    for d, g in enumerate(reps):
        s = GpuScene(h.desc, d, motion=h.motion)
        want, want_st = samples_and_counters(s, h)
        s.close()
        assert np.array_equal(got[d][0].view(np.uint32), want.view(np.uint32)), (d, np.argwhere(got[d][0] != want)[:5])
        assert got[d][1] == want_st, d
        assert want_st["rays"] > 0
    for g in reps:
        g.close()


def test_render_multi_over_replicas():
    h = scenes.cornell_box(xres=24, yres=16, spp=4, materials="mixed", n_threads=1)
    reps = create_multi(h.desc, list(range(N_ALL)))
    singles = [GpuScene(h.desc, d) for d in range(N_ALL)]
    a, sa = render_multi(reps, h.params)
    b, sb = render_multi(singles, h.params)
    assert (sa["rays"], sa["camera_rays"]) == (sb["rays"], sb["camera_rays"])
    assert np.allclose(a, b, rtol=2e-6, atol=1e-6)  # (the film sum adds samples with atomics: the order, hence the last bit, may vary)
    for g in reps + singles:
        g.close()


def test_destroying_one_replica_leaves_the_others_whole():
    if N_ALL < 2:
        pytest.skip("one device: there is no other replica")
    h = scenes.statue(n_side=STATUE_SIDE, xres=8, yres=8, spp=2)
    reps = create_multi(h.desc, list(range(N_ALL)))
    s = GpuScene(h.desc, N_ALL - 1)
    want = samples_and_counters(s, h)
    s.close()
    reps[0].close()  # the owner of slice 0 of every array
    for g in reps[1:]:
        got = samples_and_counters(g, h)
        assert np.array_equal(got[0].view(np.uint32), want[0].view(np.uint32)) and got[1] == want[1]
    for g in reversed(reps[1:]):
        g.close()


def test_each_large_array_crosses_pcie_once():
    """scene_bytes of a replica = the bytes its device received from the host.  The statue has no textures, so its large arrays are
    exactly the caller's nodes, triangle records and per-vertex attributes; everything else is the small tables every device gets."""
    h = scenes.statue(n_side=STATUE_SIDE, xres=8, yres=8, spp=2)
    d = h.desc.contents
    big = 32 * d.n_nodes + 24 * d.n_tris
    for i in range(d.n_meshes):
        m = d.meshes[i]
        big += m.n_verts * (12 + (12 if m.n else 0) + (8 if m.uv else 0) + (12 if m.s else 0))
    s = GpuScene(h.desc, 0)
    one = s.upload_bytes()
    s.close()
    small = one - big
    assert small > 0
    reps = create_multi(h.desc, list(range(N_ALL)))
    got = [g.upload_bytes() for g in reps]
    for g in reps:
        g.close()
    if peer_everywhere(N_ALL):
        assert sum(got) == one + (N_ALL - 1) * small, (got, one, small)
        assert all(abs((x - small) - big / N_ALL) <= 128 for x in got), got  # slices of whole elements: each within one element of 1/n
    elif EMULATED:  # no pair has peer access: every device uploads every slice itself
        assert got == [one] * N_ALL, (got, one)
    else:
        assert one * N_ALL >= sum(got) >= one + (N_ALL - 1) * small, (got, one, small)
