"""The realistic camera on the GPU: every integrator, both samplers, textures with a bump map, an animated camera, a crop window, a
heavily vignetting lens, both weighting modes, render_multi over replicas and statue tiles, against the oracle extended by an
independently written RealisticCamera (tests/lens_ref): samples, camera ray weights (through the film), film and the ray / node /
triangle counters, bit for bit.  Also run on the CPU through the kernel emulation (test_emu_realistic.py)."""
import os

import numpy as np
import pytest

import lens_ref
from rs_pbrt_b200 import GpuScene, _abi, create_multi, render_multi, scenes

pytestmark = pytest.mark.gpu
EMULATED = bool(os.environ.get("RS_PBRT_B200_LIB"))
COUNTERS = ("camera_rays", "rays", "closest_rays", "shadow_rays", "light_tri_tests", "nodes_visited", "tris_tested")


def _motion_camera(h):
    m = h.motion
    return m.contents.camera.contents if m is not None and bool(m.contents.camera) else None


def reference(h, rect=None):
    return lens_ref.LensScene(h.desc, h.camera_model, h.lens, _motion_camera(h)).render(h.params, rect)


def gpu_samples(g, h, rect):
    rp = h.params.contents
    old = rp.flags
    rp.flags = old | _abi.RENDER_COUNT_WORK
    try:
        return g.render_samples(h.params, rect)
    finally:
        rp.flags = old


def assert_film(film, rfilm):
    assert np.array_equal(film[..., 3], rfilm[..., 3])
    num = float(np.sum((film[..., :3].astype(np.float64) - rfilm[..., :3]) ** 2))
    den = float(np.sum(rfilm[..., :3].astype(np.float64) ** 2))
    assert num <= 1e-10 * den, (num, den)


def compare(h):
    """GPU samples and counters equal the lens reference's; the film equals the reference's sum of L * weight * filter weight."""
    g = GpuScene(h.desc, motion=h.motion, camera=h.camera_model, lens=h.lens)
    rect = list(h.params.contents.sample_bounds)
    got, gst = gpu_samples(g, h, rect)
    film, fst = g.render(h.params)
    g.close()
    rfilm, ref, weights, rst = reference(h, rect)
    assert np.array_equal(got.view(np.uint32), ref.reshape(got.shape).view(np.uint32)), np.argwhere(got != ref.reshape(got.shape))[:5]
    for k in COUNTERS:
        assert gst[k] == rst[k], (k, gst[k], rst[k])
    for k in ("camera_rays", "rays", "closest_rays", "shadow_rays"):
        assert fst[k] == rst[k], (k, fst[k], rst[k])
    assert_film(film, rfilm)
    return weights, rst


CASES = [
    dict(),                                                      # path, Sobol'
    dict(sampler="halton"),
    dict(integrator=("ao", 8, True)),
    dict(integrator=("direct", "all"), lights="delta"),
    dict(integrator=("direct", "one"), materials="mixed"),
    dict(integrator="whitted", materials="mixed"),
    dict(textures="ewa"),
    dict(textures="trilinear", sampler="halton"),
    dict(textures="ewa+float+graph+bump"),
    dict(textures="ewa", integrator=("direct", "all")),
    dict(crop=[0.2, 0.85, 0.1, 0.7]),
    dict(simpleweighting=False, shutter=(0.1, 0.8)),
]


def _id(c):
    return ",".join("%s=%s" % kv for kv in c.items()) or "default"


@pytest.mark.parametrize("kw", CASES, ids=[_id(c) for c in CASES])
def test_realistic_camera_matches_the_reference(kw):
    compare(scenes.cornell_box(**dict(dict(xres=20, yres=14, spp=8, n_threads=1, camera="realistic"), **kw)))


@pytest.mark.parametrize("kw", [dict(), dict(integrator=("ao", 4, True)), dict(textures="ewa", integrator="whitted", materials="mixed")],
                         ids=["path", "ao", "ewa-whitted"])
def test_vignetting_lens_matches_the_reference(kw):
    """A film twice the lens's image circle: the corners vignette (weight 0, L = 0, no ray traced, the filter weight still counted)."""
    h = scenes.cornell_box(xres=20, yres=14, spp=8, n_threads=1, camera="realistic", filmdiagonal=90.0, **kw)
    weights, rst = compare(h)
    n = weights.size
    assert (weights == 0).sum() > n // 8 and rst["camera_rays"] == (weights > 0).sum() < n
    assert weights[0, 0].max() == 0.0 and weights[-1, -1].max() == 0.0  # black corners


@pytest.mark.parametrize("kw", [dict(), dict(textures="ewa", sampler="halton")], ids=["path", "ewa-halton"])
def test_animated_camera_matches_the_reference(kw):
    h = scenes.motion_cornell(xres=18, yres=12, spp=8, dolly=120.0, pan=15.0, n_threads=1, camera="realistic", **kw)
    assert _motion_camera(h) is not None
    compare(h)


def test_render_multi_over_replicas():
    """render_multi over replicas from pbrt_gpu_scene_create_lens (every device there is) gives the reference's film."""
    if EMULATED:
        n = int(os.environ.get("PB_EMU_DEVICES", "1"))
    else:
        import torch

        n = torch.cuda.device_count()
    h = scenes.cornell_box(xres=20, yres=14, spp=8, n_threads=1, camera="realistic", textures="ewa", materials="mixed")
    reps = create_multi(h.desc, list(range(n)), motion=h.motion, camera=h.camera_model, lens=h.lens)
    film, st = render_multi(reps, h.params)
    for g in reps:
        g.close()
    rfilm, _, _, rst = reference(h)
    for k in ("camera_rays", "rays", "closest_rays", "shadow_rays"):
        assert st[k] == rst[k], (k, st[k], rst[k])
    assert_film(film, rfilm)


def test_statue_tiles_at_full_sample_count():
    """Four scattered 8x8 tiles of the statue at its benchmark sample count (128; 16 in the emulation), bit for bit."""
    side, spp = (40, 16) if EMULATED else (160, 128)
    h = scenes.statue(n_side=side, xres=64, yres=64, spp=spp, n_threads=4, camera="realistic")
    g = GpuScene(h.desc, camera=h.camera_model, lens=h.lens)
    ref = lens_ref.LensScene(h.desc, h.camera_model, h.lens)
    for x0, y0 in [(8, 16), (40, 8), (24, 40), (48, 48)]:
        rect = [x0, y0, x0 + 8, y0 + 8]
        got, gst = gpu_samples(g, h, rect)
        _, want, _, rst = ref.render(h.params, rect)
        want = want.reshape(got.shape)
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (rect, np.argwhere(got != want)[:5])
        for k in COUNTERS:
            assert gst[k] == rst[k], (rect, k, gst[k], rst[k])
    g.close()


def test_known_answer_rays():
    """pbrt_gpu_kat_realistic_rays: the device's generate_ray_differential equals the reference's over random camera samples
    (10^6; 2 * 10^4 in the emulation), vignetted ones included, animated camera included."""
    n = 20000 if EMULATED else 1000000
    rng = np.random.default_rng(7)
    for h in (scenes.cornell_box(xres=32, yres=24, spp=1, n_threads=1, camera="realistic", filmdiagonal=60.0),
              scenes.motion_cornell(xres=32, yres=24, spp=1, dolly=120.0, pan=15.0, n_threads=1, camera="realistic")):
        res = h.camera_model.contents.full_resolution
        pf = (rng.random((n, 2)) * np.array([res[0], res[1]])).astype(np.float32)
        pl = rng.random((n, 2)).astype(np.float32)
        t = rng.random(n).astype(np.float32)
        g = GpuScene(h.desc, motion=h.motion, camera=h.camera_model, lens=h.lens)
        got = g.kat_realistic_rays(pf, pl, t)
        g.close()
        want = lens_ref.camera_rays(h.desc.contents.camera, h.lens, h.camera_model, pf, pl, t, _motion_camera(h))
        assert 0 < (want["weight"] == 0).sum() < n or h.motion is not None
        for k in want:
            assert np.array_equal(got[k].view(np.uint32), want[k].view(np.uint32)), (k, np.argwhere(got[k] != want[k])[:5])
