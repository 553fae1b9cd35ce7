"""Orthographic and environment cameras on the GPU: every integrator, both samplers, thin lens, textures, an animated camera, a crop
window, render_multi over replicas and a statue tile set, against the oracle extended by independently written cameras
(tests/camera_ref), sample for sample and bit for bit, with the ray / node / triangle counters.  Also run on the CPU through the
kernel emulation (test_emu_cameras.py)."""
import os

import numpy as np
import pytest

import camera_ref
from rs_pbrt_b200 import GpuScene, _abi, create_multi, render_multi, scenes

pytestmark = pytest.mark.gpu
EMULATED = bool(os.environ.get("RS_PBRT_B200_LIB"))
COUNTERS = ("camera_rays", "rays", "closest_rays", "shadow_rays", "light_tri_tests", "nodes_visited", "tris_tested")


def _motion_camera(h):
    m = h.motion
    return m.contents.camera.contents if m is not None and bool(m.contents.camera) else None


def reference(h, rect=None):
    return camera_ref.CameraScene(h.desc, h.camera_model, _motion_camera(h)).render(h.params, rect)


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
    """GPU samples and counters equal the camera reference's; the film equals the sum of the reference's samples."""
    g = GpuScene(h.desc, motion=h.motion, camera=h.camera_model)
    rect = list(h.params.contents.sample_bounds)
    got, gst = gpu_samples(g, h, rect)
    film, fst = g.render(h.params)
    g.close()
    rfilm, ref, _, rst = reference(h, rect)
    assert np.array_equal(got.view(np.uint32), ref.view(np.uint32)), np.argwhere(got != ref)[:5]
    for k in COUNTERS:
        assert gst[k] == rst[k], (k, gst[k], rst[k])
    for k in ("camera_rays", "rays", "closest_rays", "shadow_rays"):
        assert fst[k] == rst[k], (k, fst[k], rst[k])
    assert_film(film, rfilm)
    return got


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
    dict(textures="ewa", integrator=("direct", "all")),          # the direct kernels' camera-ray differential (or its absence)
    dict(textures="trilinear", integrator="whitted", materials="mixed"),
    dict(crop=[0.2, 0.85, 0.1, 0.7]),                            # sample bounds != full resolution
    dict(crop=[0.3, 0.9, 0.25, 0.8], textures="ewa"),
]
ORTHO_ONLY = [
    dict(lensradius=40.0, focaldistance=900.0),                  # thin lens
    dict(lensradius=40.0, focaldistance=900.0, textures="ewa"),  # the lens differential that aims both rays at one focus point
    dict(lensradius=25.0, focaldistance=700.0, textures="trilinear", integrator="whitted", materials="mixed"),
]


def _id(c):
    return ",".join("%s=%s" % kv for kv in c.items()) or "default"


@pytest.mark.parametrize("kind", ["orthographic", "environment"])
@pytest.mark.parametrize("kw", CASES, ids=[_id(c) for c in CASES])
def test_camera_matches_the_reference(kind, kw):
    kw = dict(dict(xres=20, yres=14, spp=8, n_threads=1, camera=kind), **kw)
    compare(scenes.cornell_box(**kw))


@pytest.mark.parametrize("kw", ORTHO_ONLY, ids=[_id(c) for c in ORTHO_ONLY])
def test_orthographic_thin_lens_matches_the_reference(kw):
    compare(scenes.cornell_box(xres=20, yres=14, spp=8, n_threads=1, camera="orthographic", **kw))


@pytest.mark.parametrize("kind", ["orthographic", "environment"])
@pytest.mark.parametrize("kw", [dict(), dict(textures="ewa", sampler="halton"), dict(integrator=("direct", "one")), dict(shutter=(0.2, 0.7))],
                         ids=["path", "ewa-halton", "direct-one", "shutter"])
def test_animated_camera_matches_the_reference(kind, kw):
    h = scenes.motion_cornell(xres=18, yres=12, spp=8, dolly=120.0, pan=15.0, n_threads=1, camera=kind, **kw)
    assert _motion_camera(h) is not None
    compare(h)


def test_environment_camera_reaches_the_shutter_times():
    """ray.time = lerp(sample.time, shutter_open, shutter_close) through the animated camera: the reference's ray times span the
    shutter and the GPU's samples equal the reference's."""
    h = scenes.motion_cornell(xres=12, yres=8, spp=8, dolly=120.0, pan=30.0, shutter=(0.25, 0.75), n_threads=1, camera="environment")
    _, _, times, _ = reference(h)
    assert times.min() >= 0.25 and times.max() <= 0.75 and times.max() - times.min() > 0.4
    compare(h)


@pytest.mark.parametrize("kind", ["orthographic", "environment"])
def test_render_multi_over_replicas(kind):
    """render_multi over replicas from pbrt_gpu_scene_create_camera (every device there is) gives the reference's film."""
    if EMULATED:
        n = int(os.environ.get("PB_EMU_DEVICES", "1"))
    else:
        import torch

        n = torch.cuda.device_count()
    h = scenes.cornell_box(xres=20, yres=14, spp=8, n_threads=1, camera=kind, textures="ewa", materials="mixed")
    reps = create_multi(h.desc, list(range(n)), motion=h.motion, camera=h.camera_model)
    film, st = render_multi(reps, h.params)
    for g in reps:
        g.close()
    rfilm, _, _, rst = reference(h)
    for k in ("camera_rays", "rays", "closest_rays", "shadow_rays"):
        assert st[k] == rst[k], (k, st[k], rst[k])
    assert_film(film, rfilm)


@pytest.mark.parametrize("kind", ["orthographic", "environment"])
def test_statue_tiles_at_full_sample_count(kind):
    """Four scattered 8x8 tiles of the statue at its benchmark sample count (128; 16 in the emulation), bit for bit."""
    side, spp = (40, 16) if EMULATED else (160, 128)
    h = scenes.statue(n_side=side, xres=64, yres=64, spp=spp, n_threads=4, camera=kind)
    g = GpuScene(h.desc, camera=h.camera_model)
    ref = camera_ref.CameraScene(h.desc, h.camera_model)
    for x0, y0 in [(8, 16), (40, 8), (24, 40), (48, 48)]:
        rect = [x0, y0, x0 + 8, y0 + 8]
        got, gst = gpu_samples(g, h, rect)
        _, want, _, rst = ref.render(h.params, rect)
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (rect, np.argwhere(got != want)[:5])
        for k in COUNTERS:
            assert gst[k] == rst[k], (rect, k, gst[k], rst[k])
    g.close()


def test_explicit_perspective_model_renders_like_the_plain_scene():
    """camera == NULL, an explicit perspective model and pbrt_gpu_scene_create give the same samples."""
    h = scenes.cornell_box(xres=12, yres=10, spp=4, n_threads=1, textures="ewa")
    rect = list(h.params.contents.sample_bounds)
    model = _abi.PbrtCameraModel(_abi.PBRT_CAMERA_PERSPECTIVE, (12, 10))
    a, sa = GpuScene(h.desc).render_samples(h.params, rect)
    b, sb = GpuScene(h.desc, camera=model).render_samples(h.params, rect)
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
    assert {k: sa[k] for k in COUNTERS} == {k: sb[k] for k in COUNTERS}
