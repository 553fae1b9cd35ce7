"""Motion blur on the GPU: an animated camera under every integrator and sampler, against the oracle extended by an independently
written AnimatedTransform (tests/motion_ref), sample for sample and bit for bit, and against the float64 closed forms of
tests/motion_scenes.py.  Also run on the CPU through the kernel emulation (test_emu_motion.py)."""
import ctypes as C
import os

import numpy as np
import pytest

import motion_ref
import motion_scenes
from rs_pbrt_b200 import GpuScene, _abi, pbrt_export, scenes

pytestmark = pytest.mark.gpu
EMULATED = bool(os.environ.get("RS_PBRT_B200_LIB"))


def compare_motion(h, res_check=True):
    """GPU samples and ray counters equal the motion reference's; the film equals the sum of the samples the reference made."""
    motion = h.motion
    assert motion is not None and bool(motion.contents.camera)
    g = GpuScene(h.desc, motion=motion)
    rect = list(h.params.contents.sample_bounds)
    got, gst = g.render_samples(h.params, rect)
    film, gfst = g.render(h.params)
    g.close()
    rfilm, ref, _, rst = motion_ref.MotionScene(h.desc, motion.contents.camera.contents).render(h.params, rect)
    assert np.array_equal(got.view(np.uint32), ref.view(np.uint32)), np.argwhere(got != ref)[:5]
    for k in ("camera_rays", "closest_rays", "shadow_rays"):
        assert gst[k] == rst[k] == gfst[k], (k, gst[k], rst[k], gfst[k])
    assert np.array_equal(film[..., 3], rfilm[..., 3])
    num = float(np.sum((film[..., :3].astype(np.float64) - rfilm[..., :3]) ** 2))
    den = float(np.sum(rfilm[..., :3].astype(np.float64) ** 2))
    assert num <= 1e-10 * den, (num, den)
    return got


CASES = [
    dict(),                                                            # dolly and pan, Sobol', pinhole, path
    dict(dolly=0.0, pan=25.0, lensradius=8.0, focaldistance=800.0),   # rotation only (slerp), thin lens
    dict(sampler="halton", shutter=(0.1, 0.6)),
    dict(textures="ewa", pan=-10.0),                                   # ray differentials through the interpolated camera
    dict(integrator=("ao", 8, True)),
    dict(integrator=("direct", "all"), lights="delta"),
    dict(integrator=("direct", "one"), materials="mixed"),
    dict(integrator="whitted", materials="mixed"),
    dict(shutter=(-0.5, 1.5), transform_times=(0.2, 0.8)),             # shutter wider than TransformTimes: clamped keyframes
    dict(dolly=60.0, pan=200.0),                                       # keyframe quaternions in opposite hemispheres: the r[1] flip
]


def _pre_flip_dot(at):
    """quat_dot of the two keyframes' rotations as decompose gives them, before AnimatedTransform::new flips r[1]."""
    q0 = motion_ref.decompose(np.array(at.start, np.float32).reshape(4, 4))[1]
    q1 = motion_ref.decompose(np.array(at.end, np.float32).reshape(4, 4))[1]
    return float(np.dot(q0.astype(np.float64), q1))


def test_the_flip_case_needs_the_flip():
    h = scenes.motion_cornell(xres=8, yres=8, spp=1, dolly=60.0, pan=200.0, n_threads=1)
    assert _pre_flip_dot(h.motion.contents.camera.contents) < 0


@pytest.mark.parametrize("kw", CASES, ids=[",".join("%s=%s" % kv for kv in c.items()) or "default" for c in CASES])
def test_animated_camera_matches_the_reference(kw):
    kw = dict(dict(xres=20, yres=16, spp=8, dolly=150.0, pan=12.0), **kw)
    compare_motion(scenes.motion_cornell(n_threads=1, **kw))


def test_equal_keyframes_render_like_a_static_camera():
    h = scenes.cornell_box(xres=16, yres=16, spp=4, n_threads=1)
    c2w = np.array(h.desc.contents.camera.camera_to_world, np.float32).reshape(4, 4)
    at = motion_ref.animated_transform(c2w, c2w)
    md = _abi.PbrtMotionDesc()
    md.camera = C.pointer(at)
    rect = list(h.params.contents.sample_bounds)
    a, _ = GpuScene(h.desc, motion=md).render_samples(h.params, rect)
    b, _ = GpuScene(h.desc).render_samples(h.params, rect)
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32))


HUNT = int(os.environ.get("RS_PBRT_MOTION_HUNT", "12"))


@pytest.mark.parametrize("seed", range(HUNT))
def test_random_camera_keyframes_match_the_reference(seed):
    """Random end keyframes (eye moved up to 250 units, view turned by up to 300 degrees about a random tilted axis), random
    TransformTimes and shutter, either sampler and integrator path or directlighting.  RS_PBRT_MOTION_HUNT sets the number of draws."""
    rng = np.random.default_rng(1000 + seed)
    eye = np.array([278.0, 273.0, -800.0]) + rng.uniform(-250, 250, 3)
    ax = rng.normal(size=3)
    from scipy.spatial.transform import Rotation
    d = Rotation.from_rotvec(ax / np.linalg.norm(ax) * np.radians(rng.uniform(-300, 300))).apply([0.0, 0.0, 1.0])
    up = [0.0, 1.0, 0.0] if abs(d[1]) < 0.95 else [1.0, 0.0, 0.0]
    t0 = float(rng.uniform(-0.5, 0.5))
    times = (t0, t0 + float(rng.uniform(0.1, 2.0)))
    s0 = t0 + float(rng.uniform(-0.3, 0.2))  # the shutter opens near the start keyframe, which looks into the box
    shutter = (s0, s0 + float(rng.uniform(0.0, 2.0)))
    h = scenes.cornell_box(xres=12, yres=10, spp=4, n_threads=1, camera_end=scenes.look_at_matrix(eye, eye + 800.0 * d, up), shutter=shutter,
                           transform_times=times, sampler=["sobol", "halton"][seed % 2],
                           integrator=["path", ("direct", "all")][(seed // 2) % 2], lensradius=[0.0, 5.0][(seed // 4) % 2], focaldistance=800.0)
    assert np.any(compare_motion(h) > 0)


@pytest.mark.parametrize("shutter", [(0.25, 0.75), (-0.5, 1.5)])
def test_panning_camera_against_the_closed_form(shutter):
    _closed_form(dict(shutter=shutter))


def test_turning_camera_against_the_closed_form():
    _closed_form(dict(x0=-0.5, x1=0.8, yaw=(20.0, -25.0), shutter=(0.1, 0.9)))


def _closed_form(kw):
    shutter = kw["shutter"]
    h = motion_scenes.pan_scene(xres=16, yres=8, spp=8, **kw)
    g = GpuScene(h.desc, motion=h.motion)
    got, _ = g.render_samples(h.params, list(h.params.contents.sample_bounds))
    import oracle_lib
    o = oracle_lib.OracleScene(h.desc)
    checked = 0
    for py in range(8):
        for px in range(16):
            for s in range(8):
                cs = o.camera_sample(h.params, px, py, s)
                exp, edge = motion_scenes.pan_radiance(cs[None, 0:2], cs[2], 16, 8, **kw)
                if edge[0] < 2e-3:
                    continue
                checked += 1
                assert np.all(np.abs(got[py, px, s] - exp[0]) <= 1e-4 * max(exp[0], 1e-3)), (px, py, s, got[py, px, s], exp[0])
    assert checked > 900


def _kat_keyframes():
    """Seven transforms, drawn from their own generator so that they are the same whatever number of times is tested: the slerp's lerp
    branch, an ordinary and a wide rotation, two pairs whose quaternions (as decompose returns them) lie in opposite hemispheres (the
    r[1] flip; the test checks that they do), a negative rotation and translation / scale only."""
    from scipy.spatial.transform import Rotation

    rng = np.random.default_rng(7)
    out = []
    # flip: q0 = identity (w = 1), and Quaternion::new makes the largest component of the end rotation's positive (trace <= 0), which
    # for these angle / axis-sign pairs leaves w < 0
    for span, flip, sign in [(0.01, False, 0), (0.5, False, 0), (2.0, False, 0), (3.6, True, 1), (2.6, True, -1), (-2.5, False, 0), (0.0, False, 0)]:
        ax = rng.normal(size=3)
        ax = (sign * np.abs(ax) if sign else ax) / np.linalg.norm(ax)
        a0 = 0.0 if flip else rng.uniform(-3, 3)

        def key(angle):
            M = np.eye(4)
            M[:3, :3] = Rotation.from_rotvec(ax * angle).as_matrix() @ np.diag(rng.uniform(0.5, 2, 3))
            M[:3, 3] = rng.uniform(-4, 4, 3)
            return M
        out.append((motion_ref.animated_transform(key(a0), key(a0 + span), -0.5, 2.0), flip))
    return out


def test_kat_animated_interpolate_is_bit_equal_to_the_reference():
    L = _abi.load()
    n = 10 ** 4 if EMULATED else 10 ** 6
    fp = lambda a: a.ctypes.data_as(C.POINTER(C.c_float))
    rng = np.random.default_rng(8)
    for k, (at, flip) in enumerate(_kat_keyframes()):
        assert (_pre_flip_dot(at) < 0) == flip, (k, _pre_flip_dot(at))
        t = rng.uniform(-1.0, 2.5, n).astype(np.float32)
        t[:4] = [-0.5, 2.0, np.nextafter(np.float32(-0.5), np.float32(1)), np.nextafter(np.float32(2.0), np.float32(0))]
        m, mi = np.zeros((n, 16), np.float32), np.zeros((n, 16), np.float32)
        assert L.pbrt_gpu_kat_animated_interpolate(0, C.byref(at), n, fp(t), fp(m), fp(mi)) == 0
        rm, rmi = motion_ref.interpolate(at, t)
        assert np.array_equal(m.view(np.uint32), rm.reshape(n, 16).view(np.uint32)), k
        assert np.array_equal(mi.view(np.uint32), rmi.reshape(n, 16).view(np.uint32)), k


def test_pbrt_export_writes_the_camera_motion(tmp_path):
    h = scenes.motion_cornell(xres=16, yres=16, spp=4, shutter=(0.1, 0.7), transform_times=(0.0, 2.0), n_threads=1)
    pbrt_export.write(h, tmp_path / "motion.pbrt")
    text = (tmp_path / "motion.pbrt").read_text()
    for s in ("TransformTimes 0.0 2.0", "ActiveTransform StartTime", "ActiveTransform EndTime", "ActiveTransform All", '"float shutteropen" [0.1'):
        assert s in text, s
    assert text.index("ActiveTransform EndTime") < text.index("Camera ")
    # read the keyframes back as rs_pbrt does: `Transform` takes the matrix column-major (the transpose of the row-major m[r][c]), the
    # CTM at the Camera directive is world_to_camera, and camera_to_world = its inverse (api.rs:497-502)
    lines = text.splitlines()
    i = lines.index("ActiveTransform EndTime")
    w2c_end = np.array([float(v) for v in lines[i + 1].split("[")[1].split("]")[0].split()], np.float64).reshape(4, 4).T
    end = np.array(h.motion.contents.camera.contents.end, np.float64).reshape(4, 4)
    assert np.abs(np.linalg.inv(w2c_end) - end).max() <= 1e-5 * np.abs(end).max()
    look = lines[lines.index("ActiveTransform StartTime") + 1].split()
    assert look[0] == "LookAt" and [float(v) for v in look[1:4]] == [278.0, 273.0, -800.0]
    shut = text.split('"float shutteropen" [')[1]
    assert float(shut.split("]")[0]) == np.float32(0.1) and float(shut.split('"float shutterclose" [')[1].split("]")[0]) == np.float32(0.7)
