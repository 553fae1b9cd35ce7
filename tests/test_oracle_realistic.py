"""The realistic camera's construction and ray generation held to float64 closed forms that share no code with what they test.

The host mirror's RealisticCamera::new (pbrt_host_camera_realistic: units, aperture clamp, focus_thick_lens, exit-pupil bounds) and the
reference restatement the GPU is compared with bit for bit (tests/lens_ref) are checked against: a float64 vector Snell's-law tracer
over a singlet and a 50 mm double-Gauss; the focus from paraxial ABCD matrices; the pupil bounds of a stop-only lens and of a two-stop
lens whose off-axis pupil is a disk away from the axis (the reference's zero-box start puts the axis inside every bin); both weightings;
and the export of the camera to a .pbrt file and its lens file, read back."""
import ctypes as C

import numpy as np
import pytest
from scipy.optimize import brentq

import lens_ref
from rs_pbrt_b200 import HostScene, _abi, scenes

SINGLET = [[50.0, 5.0, 1.5, 20.0], [-50.0, 45.0, 1.0, 20.0]]  # biconvex, n = 1.5, R = 50 mm; the last thickness is then focused


def _elements(h):
    L = h.lens.contents
    return np.array([[L.elements[i].curvature_radius, L.elements[i].thickness, L.elements[i].eta, L.elements[i].aperture_radius]
                     for i in range(L.n_elements)], np.float64)


def _bounds(h):
    return np.array([h.lens.contents.exit_pupil_bounds[i] for i in range(256)], np.float64).reshape(64, 4)


def _scene(lens, **kw):
    return scenes.cornell_box(xres=24, yres=16, spp=1, n_threads=1, camera="realistic", lensfile=lens, **kw)


def _identity_camera(shutter=(0.0, 1.0)):
    cam = _abi.PbrtCamera()
    for i in range(4):
        cam.camera_to_world[5 * i] = 1.0
        cam.raster_to_camera[5 * i] = 1.0
    cam.shutter_open, cam.shutter_close = shutter
    return cam


def _eta(e):
    return 1.0 if e == 0.0 else e


def snell_trace(el, p, d):
    """Float64 vector Snell's law through the lens `el` (metres, scene side first) from camera-space point p along d (towards +z):
    -> (exit point, exit direction), or None when a surface is missed, an aperture clips or the ray reflects totally."""
    z = np.cumsum(el[::-1, 1])[::-1]  # camera-space z of each interface's vertex (the last thickness is the lens-film distance)
    p, d = np.array(p, np.float64), np.array(d, np.float64) / np.linalg.norm(d)
    for i in range(len(el) - 1, -1, -1):
        R, _, _, a = el[i]
        if R == 0.0:  # the stop: a plane
            t = (z[i] - p[2]) / d[2]
            q = p + t * d
        else:
            c = np.array([0.0, 0.0, z[i] - R])
            oc = p - c
            b = np.dot(oc, d)
            disc = b * b - (np.dot(oc, oc) - R * R)
            if disc < 0:
                return None
            ts = [-b - np.sqrt(disc), -b + np.sqrt(disc)]
            q = None
            for t in sorted(ts):  # the cap of the sphere that holds the vertex
                qq = p + t * d
                if t >= 0 and np.sign(qq[2] - c[2]) == np.sign(R):
                    q = qq
                    break
            if q is None:
                return None
        if q[0] ** 2 + q[1] ** 2 > a * a:
            return None
        p = q
        if R != 0.0:
            n = (q - c) / abs(R)
            if np.dot(n, d) > 0:
                n = -n
            mu = _eta(el[i, 2]) / (_eta(el[i - 1, 2]) if i > 0 else 1.0)
            cos_i = -np.dot(n, d)
            sin2_t = mu * mu * (1.0 - cos_i * cos_i)
            if sin2_t >= 1.0:
                return None
            d = mu * d + (mu * cos_i - np.sqrt(1.0 - sin2_t)) * n
            d /= np.linalg.norm(d)
    return p, d


def camera_sample_f64(el, bounds, diag, res, p_film, p_lens, simple=True, shutter=(0.0, 1.0)):
    """generate_ray's film point, exit-pupil point and weight in float64 (realistic.rs:198-251,656-688; film.rs:293-307)."""
    aspect = res[1] / res[0]
    x = np.sqrt(diag * diag / (1 + aspect * aspect))
    y = aspect * x
    fx = -(-x / 2 + (x / 2 - -x / 2) * p_film[0] / res[0])
    fy = -y / 2 + (y / 2 - -y / 2) * p_film[1] / res[1]
    r = np.hypot(fx, fy)
    b = bounds[min(63, int(np.floor(r / (diag / 2) * 64)))]
    lx, ly = b[0] + (b[2] - b[0]) * p_lens[0], b[1] + (b[3] - b[1]) * p_lens[1]
    s, c = (fy / r, fx / r) if r != 0 else (0.0, 1.0)
    rear = np.array([c * lx - s * ly, s * lx + c * ly, el[-1, 1]])
    film = np.array([fx, fy, 0.0])
    dd = rear - film
    cos4 = (dd[2] / np.linalg.norm(dd)) ** 4
    area = (b[2] - b[0]) * (b[3] - b[1])
    w = cos4 * area / ((bounds[0, 2] - bounds[0, 0]) * (bounds[0, 3] - bounds[0, 1])) if simple else \
        (shutter[1] - shutter[0]) * cos4 * area / el[-1, 1] ** 2
    return film, dd, w


@pytest.mark.parametrize("lens,kw", [(SINGLET, dict(focusdistance=1000.0)), (scenes.DGAUSS_50MM, dict(aperturediameter=8.0)),
                                     (scenes.DGAUSS_50MM, dict(aperturediameter=17.0, simpleweighting=False, shutter=(0.2, 0.7)))],
                         ids=["singlet", "dgauss-f6", "dgauss-open-nonsimple"])
def test_lens_rays_and_weights_match_a_float64_snell_tracer(lens, kw):
    """lens_ref's generate_ray (what the GPU equals bit for bit) against the float64 tracer: the same samples pass, and the exit point,
    direction and weight agree to float32 accuracy (2e-6 m, 2e-5, 2e-5 relative)."""
    h = _scene(lens, **kw)
    el, bounds = _elements(h), _bounds(h)
    L = h.lens.contents
    res = tuple(h.camera_model.contents.full_resolution)
    shutter = kw.get("shutter", (0.0, 1.0))
    rng = np.random.default_rng(3)
    n = 4000
    pf = (rng.random((n, 2)) * np.array(res)).astype(np.float32)
    pl = rng.random((n, 2)).astype(np.float32)
    got = lens_ref.camera_rays(_identity_camera(shutter), h.lens, h.camera_model, pf, pl, np.zeros(n, np.float32))
    agree = passed = 0
    for k in range(n):
        film, dd, w = camera_sample_f64(el, bounds, float(L.film_diagonal), res, pf[k].astype(np.float64), pl[k].astype(np.float64),
                                        simple=bool(L.simple_weighting), shutter=shutter)
        ref = snell_trace(el, film, dd)
        f32_pass = got["weight"][k] != 0.0
        # the shifted rays can zero a weight whose main ray passes: compare the main ray only where f32 kept the sample
        if f32_pass:
            assert ref is not None, k
            passed += 1
            np.testing.assert_allclose(got["o"][k], ref[0], atol=2e-6)
            np.testing.assert_allclose(got["d"][k], ref[1], atol=2e-5)
            np.testing.assert_allclose(got["weight"][k], w, rtol=2e-5)
        agree += (ref is not None) == f32_pass
    assert passed > n // 4 and agree >= 0.99 * n, (passed, agree)


def paraxial(el, n_skip_last=True):
    """ABCD of the lens from the first vertex to the last (ray vector (y, n u)), float64."""
    M = np.eye(2)
    for i in range(len(el)):
        R, t, eta, _ = el[i]
        n1, n2 = (_eta(el[i - 1, 2]) if i > 0 else 1.0), _eta(eta)
        if R != 0.0:
            M = np.array([[1.0, 0.0], [-(n2 - n1) / R, 1.0]]) @ M
        if i < len(el) - 1:
            M = np.array([[1.0, t / n2], [0.0, 1.0]]) @ M
    return M


@pytest.mark.parametrize("lens,focus", [(SINGLET, 1000.0), (SINGLET, 2.0), (scenes.DGAUSS_50MM, 1000.0), (scenes.DGAUSS_50MM, 1.5)],
                         ids=["singlet-far", "singlet-near", "dgauss-far", "dgauss-near"])
def test_focus_thick_lens_matches_paraxial_optics(lens, focus):
    """focus_thick_lens: the film sits where the paraxial image of the plane `focusdistance` in front of the film falls (ABCD matrices,
    float64).  Tolerance: 1e-6 m for the thick-lens approximation's rays 35 um off the axis (paraxial to about (h / f)^2), plus four
    f32 spacings of focusdistance: the reference's delta = (pz1 - z + pz0 - sqrt(c)) / 2 subtracts numbers of that size in f32."""
    h = _scene(lens, focusdistance=focus, aperturediameter=8.0)
    el = _elements(h)
    M = paraxial(el)
    (A, B), (Cc, D) = M
    front = el[:-1, 1].sum()

    def residual(t_last):  # image distance behind the last vertex minus the lens-film distance
        so = focus - (front + t_last)
        return -(A * so + B) / (Cc * so + D) - t_last

    t = brentq(residual, 0.5 * el[-1, 1], 1.5 * el[-1, 1])
    assert abs(el[-1, 1] - t) < 1e-6 + 4 * float(np.spacing(np.float32(focus))), (el[-1, 1], t)
    rows = np.array(lens, np.float64)
    assert np.array_equal(el[:-1, 1], (rows[:-1, 1].astype(np.float32) * np.float32(0.001)).astype(np.float64))


def _pupil(el_m, diag):
    el = (_abi.PbrtLensElement * len(el_m))(*[_abi.PbrtLensElement(*map(float, r)) for r in el_m])
    out = np.zeros(256, np.float32)
    L = _abi.load()
    assert L.pbrt_host_lens_exit_pupil(el, len(el_m), diag, out.ctypes.data_as(C.POINTER(C.c_float))) == 0
    return out.reshape(64, 4).astype(np.float64)


def test_stop_only_lens_pupil_is_the_stop_disk():
    """One stop of radius a on the rear sampling plane: every bin's pupil is the disk |p| <= a, bounded to within the sampling grid and
    expanded by 2 |diag| / 1024 of the sampled square (realistic.rs:647-650)."""
    a, t = 0.004, 0.03
    b = _pupil([[0.0, t, 0.0, a]], 0.035)
    delta = 2.0 * np.hypot(3 * a, 3 * a) / 1024.0
    spacing = 3 * a / 512.0
    for k in range(64):
        np.testing.assert_allclose(b[k], [-a - delta, -a - delta, a + delta, a + delta], atol=spacing)


def test_two_stop_lens_off_axis_pupil_keeps_the_origin():
    """A rear stop on the sampling plane and a small front stop further out: off axis the pupil is a disk away from the optical axis,
    yet every bin's bounds contain (0, 0) -- the running box starts as Bounds2f::default(), the zero box (geometry.rs:1865), not empty."""
    t1, t0, a1, a0, diag = 0.02, 0.02, 0.02, 0.0015, 0.035
    b = _pupil([[0.0, t0, 0.0, a0], [0.0, t1, 0.0, a1]], diag)
    k = (t1 + t0) / t1  # a ray from film x through rear-plane point p reaches the front stop at x + (p - x) k
    delta = 2.0 * np.hypot(3 * a1, 3 * a1) / 1024.0
    spacing = 3 * a1 / 512.0
    for i in range(64):
        x0, x1 = i / 64 * diag / 2, (i + 1) / 64 * diag / 2
        # points p with |x + (p - x) k| <= a0: the disk of centre x (1 - 1/k) and radius a0 / k, over x in [x0, x1]
        lo, hi = x0 * (1 - 1 / k) - a0 / k, x1 * (1 - 1 / k) + a0 / k
        want = [min(lo, 0.0) - delta, -a0 / k - delta, max(hi, 0.0) + delta, a0 / k + delta]
        np.testing.assert_allclose(b[i], want, atol=spacing)
        assert b[i, 0] < 0 < b[i, 2] and b[i, 1] < 0 < b[i, 3]
    assert lo > 0.003  # the last bins' disks lie well away from the axis: the origin is in their bounds only by the quirk


def test_aperture_clamp_and_units():
    """Lens rows in mm become metres; the stop's diameter becomes aperturediameter unless that is larger than the file's (then the
    file's is kept, realistic.rs:62-72); the film diagonal goes in mm and is kept in metres."""
    for ap, want in ((4.0, 4.0), (17.1, 17.1), (40.0, 17.1)):
        h = scenes.cornell_box(xres=8, yres=6, spp=1, n_threads=1, camera="realistic", aperturediameter=ap, filmdiagonal=43.3)
        el = _elements(h)
        assert el[5, 3] == np.float32(np.float32(want) * np.float32(0.001) / np.float32(2.0))
        assert h.lens.contents.film_diagonal == np.float32(np.float32(43.3) * np.float32(0.001))


def test_host_mirror_refuses_what_the_reference_cannot_build():
    h = HostScene()
    h.film(8, 6)
    with pytest.raises(Exception):
        h.camera_realistic([[50.0, 5.0, 1.5]])  # not a multiple of four values
    with pytest.raises(Exception):
        h.camera_realistic(SINGLET, focusdistance=0.01)  # closer than the lens can focus: the reference asserts
    with pytest.raises(Exception):
        h.film_diagonal(0.0)


@pytest.mark.parametrize("kw", [dict(), dict(simpleweighting=False, shutter=(0.1, 0.6), aperturediameter=12.0, filmdiagonal=50.0)],
                         ids=["simple", "nonsimple-diag50"])
def test_export_writes_the_realistic_camera_and_reads_back(tmp_path, kw):
    """pbrt_export writes Camera "realistic" with its lens file, aperture, focus distance, weighting and shutter, and the Film diagonal;
    tests/pbrt_reader_realistic.py reads it back to the same lens, the same pupil bounds and the same reference render."""
    import pbrt_reader_realistic
    from rs_pbrt_b200 import pbrt_export

    h = scenes.cornell_box(xres=12, yres=10, spp=2, n_threads=1, camera="realistic", **kw)
    pbrt_export.write(h, tmp_path / "scene.pbrt")
    text = (tmp_path / "scene.pbrt").read_text()
    assert 'Camera "realistic"' in text and '"string lensfile" ["scene_lens.dat"]' in text and (tmp_path / "scene_lens.dat").exists()
    h2 = pbrt_reader_realistic.read(tmp_path / "scene.pbrt", n_threads=1)
    assert np.array_equal(_elements(h), _elements(h2)) and np.array_equal(_bounds(h), _bounds(h2))
    a, b = h.lens.contents, h2.lens.contents
    assert (a.film_diagonal, a.simple_weighting) == (b.film_diagonal, b.simple_weighting)
    c1, c2 = h.desc.contents.camera, h2.desc.contents.camera
    assert (c1.shutter_open, c1.shutter_close) == (c2.shutter_open, c2.shutter_close)
    assert np.array_equal(np.array(c1.camera_to_world), np.array(c2.camera_to_world))
    _, s1, w1, st1 = lens_ref.LensScene(h.desc, h.camera_model, h.lens).render(h.params)
    _, s2, w2, st2 = lens_ref.LensScene(h2.desc, h2.camera_model, h2.lens).render(h2.params)
    assert np.array_equal(s1, s2) and np.array_equal(w1, w2) and st1["rays"] == st2["rays"]
