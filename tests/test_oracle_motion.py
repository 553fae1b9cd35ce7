"""AnimatedTransform and the animated camera against float64 closed forms that share no code with the library or the motion
reference's transform code (tests/motion_ref): scipy's polar decomposition, rotation about a fixed axis, and the moving-camera
scene of tests/motion_scenes.py."""
import numpy as np
import pytest
import scipy.linalg
from scipy.spatial.transform import Rotation

import motion_ref
import motion_scenes
import oracle_lib


def _trs(rng, angle=None, axis=None):
    axis = rng.normal(size=3) if axis is None else axis
    angle = rng.uniform(-np.pi, np.pi) if angle is None else angle
    R = Rotation.from_rotvec(axis / np.linalg.norm(axis) * angle).as_matrix()
    A = rng.normal(size=(3, 3)) * 0.3
    S = np.eye(3) * rng.uniform(0.5, 2.0) + A @ A.T  # symmetric positive definite
    M = np.eye(4)
    M[:3, :3] = R @ S
    M[:3, 3] = rng.uniform(-5, 5, 3)
    return M, R, S


def test_decompose_matches_the_polar_decomposition():
    rng = np.random.default_rng(1)
    for _ in range(200):
        M, R, S = _trs(rng)
        t, q, s = motion_ref.decompose(M.astype(np.float32))
        Rq = Rotation.from_quat(q.astype(np.float64)).as_matrix()
        u, p = scipy.linalg.polar(M[:3, :3].astype(np.float32).astype(np.float64))
        assert np.allclose(t, M[:3, 3].astype(np.float32), rtol=0, atol=0)
        assert np.abs(Rq - u).max() < 2e-5, np.abs(Rq - u).max()
        assert np.abs(s[:3, :3] - p).max() < 2e-5 * max(1.0, np.abs(p).max())
        # S = R^-1 M of the whole matrix: its last column is R^-1 t, which interpolate() never reads
        assert np.array_equal(s[3], [0, 0, 0, 1]) and np.abs(s[:3, 3] - u.T @ M[:3, 3]).max() < 1e-4


def _keyframes(rng, a0, a1, axis):
    def m(angle, tr, sc):
        M = np.eye(4)
        M[:3, :3] = Rotation.from_rotvec(axis * angle).as_matrix() @ np.diag(sc)
        M[:3, 3] = tr
        return M
    tr0, tr1 = rng.uniform(-3, 3, 3), rng.uniform(-3, 3, 3)
    sc0, sc1 = rng.uniform(0.5, 2.0, 3), rng.uniform(0.5, 2.0, 3)
    return m(a0, tr0, sc0), m(a1, tr1, sc1), (tr0, tr1, sc0, sc1)


@pytest.mark.parametrize("span", [0.02, 0.8, 2.5])  # the slerp's lerp branch (cos > 0.9995), an ordinary and a wide rotation
def test_interpolate_is_rotation_about_the_fixed_axis(span):
    rng = np.random.default_rng(int(span * 100))
    for _ in range(20):
        axis = rng.normal(size=3)
        axis /= np.linalg.norm(axis)
        a0 = rng.uniform(-1, 1)
        M0, M1, (tr0, tr1, sc0, sc1) = _keyframes(rng, a0, a0 + span, axis)
        at = motion_ref.animated_transform(M0, M1, 2.0, 5.0)
        times = np.array([1.0, 2.0, 2.5, 3.1, 4.0, 4.999, 5.0, 7.0], np.float32)
        m, mi = motion_ref.interpolate(at, times)
        for k, t in enumerate(times):
            dt = np.clip((float(t) - 2.0) / 3.0, 0.0, 1.0)
            E = np.eye(4)
            E[:3, :3] = Rotation.from_rotvec(axis * (a0 + span * dt)).as_matrix() @ np.diag((1 - dt) * sc0 + dt * sc1)
            E[:3, 3] = (1 - dt) * tr0 + dt * tr1
            # the f32 keyframes carry ~1e-7 of error and the slerp / lerp branch ~1e-6 more
            assert np.abs(m[k] - E).max() < 2e-5 * max(1.0, np.abs(E).max()), (t, np.abs(m[k] - E).max())
            assert np.abs(mi[k] @ m[k] - np.eye(4)).max() < 5e-5
        # clamping: before start_time and at it the start keyframe's own bits, after end_time and at it the end keyframe's
        assert np.array_equal(m[0], np.array(at.start).reshape(4, 4)) and np.array_equal(m[1], np.array(at.start).reshape(4, 4))
        assert np.array_equal(m[-1], np.array(at.end).reshape(4, 4)) and np.array_equal(mi[-2], np.array(at.end_inv).reshape(4, 4))


def test_equal_keyframes_return_the_start_bits():
    rng = np.random.default_rng(5)
    M, _, _ = _trs(rng)
    at = motion_ref.animated_transform(M, M, 0.0, 1.0)
    m, mi = motion_ref.interpolate(at, np.linspace(-1, 2, 31))
    assert all(np.array_equal(x, np.array(at.start).reshape(4, 4)) for x in m)
    assert all(np.array_equal(x, np.array(at.start_inv).reshape(4, 4)) for x in mi)


def _per_sample(h, ref_samples, **kw):
    """Per-sample radiance against pan_radiance: p_film and the sample's time come from the sampler, nothing else."""
    p = h.params.contents
    o = oracle_lib.OracleScene(h.desc)
    xr, yr = p.cropped_pixel_bounds[2], p.cropped_pixel_bounds[3]
    bad = checked = 0
    for py in range(yr):
        for px in range(xr):
            for s in range(p.spp):
                cs = o.camera_sample(h.params, px, py, s)
                exp, edge = motion_scenes.pan_radiance(cs[None, 0:2], cs[2], xr, yr, **kw)
                if edge[0] < 2e-3:  # within the f32 camera ray's error of an edge: either answer is right
                    continue
                checked += 1
                got = ref_samples[py, px, s]
                if not np.all(np.abs(got - exp[0]) <= 1e-4 * max(exp[0], 1e-3)):
                    bad += 1
    return bad, checked


@pytest.mark.parametrize("shutter,times", [((0.25, 0.75), (0.0, 1.0)), ((0.0, 1.0), (0.0, 1.0)), ((-0.5, 1.5), (0.0, 1.0))])
def test_panning_camera_per_sample_radiance(shutter, times):
    """A camera sliding along x past a lit quad: every sample's radiance is Kd/pi L where its ray, at ray.time, hits the quad.
    The last case opens the shutter before TransformTimes begins and closes it after they end (the transform clamps)."""
    h = motion_scenes.pan_scene(xres=16, yres=8, spp=8, shutter=shutter, times=times)
    _, samples, _, st = motion_ref.MotionScene(h.desc, h.motion.contents.camera.contents).render(h.params)
    bad, checked = _per_sample(h, samples, shutter=shutter, times=times)
    assert checked > 900 and bad == 0, (bad, checked)


@pytest.mark.parametrize("yaw,x", [((-30.0, 30.0), (0.0, 0.0)), ((20.0, -25.0), (-0.5, 0.8))])
def test_turning_camera_per_sample_radiance(yaw, x):
    """The camera turns about the vertical axis (and slides): the quad sweeps across the frame at the rate of the slerp."""
    kw = dict(x0=x[0], x1=x[1], yaw=yaw, shutter=(0.1, 0.9))
    h = motion_scenes.pan_scene(xres=16, yres=8, spp=8, **kw)
    _, samples, _, _ = motion_ref.MotionScene(h.desc, h.motion.contents.camera.contents).render(h.params)
    bad, checked = _per_sample(h, samples, **kw)
    assert checked > 900 and bad == 0, (bad, checked)


def test_motion_blurred_step_edge_matches_the_space_time_coverage():
    """Pixel means across the quad's moving left and right edges against the closed-form coverage of pixel x shutter time,
    within 4 standard errors; the standard error of the total is at most 0.25 % of its expectation."""
    xr, yr, spp = 16, 16, 2048
    h = motion_scenes.pan_scene(xres=xr, yres=yr, spp=spp, half=(1.0, 10.0))
    _, samples, _, _ = motion_ref.MotionScene(h.desc, h.motion.contents.camera.contents).render(h.params)
    lum = samples[..., 0].astype(np.float64)  # (yr, xr, spp)
    Lq = motion_scenes.KD / np.pi * motion_scenes.L_LIGHT
    cov = np.array([motion_scenes.pan_coverage(px, xr, yr) for px in range(xr)])
    partial = (cov > 0.02) & (cov < 0.98)
    assert partial.sum() >= 4
    got = lum[:, partial, :].mean(axis=(0, 2))
    se = lum[:, partial, :].std(axis=(0, 2)) / np.sqrt(yr * spp)
    assert np.all(np.abs(got - Lq * cov[partial]) <= 4 * se + 1e-3 * Lq), (got, Lq * cov[partial], se)
    tot_se = np.sqrt(np.sum(lum[:, partial, :].var(axis=(0, 2)) / (yr * spp)))
    assert tot_se <= 0.0025 * np.sum(Lq * cov[partial]), (tot_se, np.sum(Lq * cov[partial]))
    assert abs(np.sum(got) - np.sum(Lq * cov[partial])) <= 4 * tot_se
