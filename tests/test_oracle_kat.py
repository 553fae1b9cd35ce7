"""CPU tests of the ORACLE: known-answer and property tests that pin it independently of the reference
(SURVEY.md section 8c: the reference holds no golden vectors for this path), plus the frozen fixtures."""
import ctypes as C
from fractions import Fraction
from pathlib import Path

import numpy as np
import pytest

from rs_pbrt_b200 import _abi, scenes

GOLD = Path(__file__).resolve().parent / "golden"


def test_gamma_and_float_stepping(oracle):
    L = oracle.load()
    eps = np.float32(2.0 ** -24)
    for n in (2, 3, 5, 6, 7):
        want = np.float32(np.float32(n) * eps) / np.float32(np.float32(1.0) - np.float32(n) * eps)
        assert L.orc_gamma(n) == want
    for v in (0.0, -0.0, 1.0, -1.0, 1e-45, 3.4e38, 123.456, -7.5e-12):
        v32 = np.float32(v)
        assert L.orc_next_float_up(float(v32)) == np.nextafter(v32, np.float32(np.inf))
        assert L.orc_next_float_down(float(v32)) == np.nextafter(v32, np.float32(-np.inf))
    assert L.orc_next_float_up(float("inf")) == float("inf")
    assert L.orc_next_float_down(float("-inf")) == float("-inf")


def test_offset_ray_origin_moves_outside_error_box(oracle):
    L = oracle.load()
    rng = np.random.default_rng(0)
    for _ in range(200):
        p = rng.uniform(-10, 10, 3).astype(np.float32)
        err = np.abs(rng.normal(size=3)).astype(np.float32) * np.float32(1e-5)
        n = rng.normal(size=3)
        n = (n / np.linalg.norm(n)).astype(np.float32)
        w = rng.normal(size=3).astype(np.float32)
        out = np.zeros(3, np.float32)
        fp = lambda a: a.ctypes.data_as(C.POINTER(C.c_float))
        L.orc_offset_ray_origin(fp(p), fp(err), fp(n), fp(w), fp(out))
        side = np.sign(np.dot(w.astype(np.float64), n))
        d = float(np.dot(np.abs(n).astype(np.float64), err))
        # moved along +-n by at least the projected error, on the side of w
        assert side * np.dot((out - p).astype(np.float64), n) >= d * 0.999


def test_sobol_dim0_is_van_der_corput(oracle):
    L = oracle.load()
    for i in [0, 1, 2, 3, 6, 100, 12345, (1 << 20) + 3]:
        rev = int("{:032b}".format(i)[::-1], 2)
        want = min(np.float32(rev) * np.float32(2.0 ** -32), np.float32(0.99999994))
        assert L.orc_sobol_sample_float(i, 0, 0) == want


def test_sobol_first_two_dims_are_a_02_sequence(oracle):
    L = oracle.load()
    for k in range(1, 9):
        n = 1 << (2 * k if 2 * k <= 10 else 10)
        pts = np.array([[L.orc_sobol_sample_float(i, 0, 0), L.orc_sobol_sample_float(i, 1, 0)] for i in range(n)])
        # every elementary interval of area 1/n holds exactly one point
        m = int(np.log2(n))
        for a in range(m + 1):
            cx, cy = 1 << a, 1 << (m - a)
            cells = (np.floor(pts[:, 0] * cx).astype(int) * cy + np.floor(pts[:, 1] * cy).astype(int))
            assert len(np.unique(cells)) == n


@pytest.mark.parametrize("m", [1, 3, 5, 7])
def test_sobol_interval_to_index_maps_back_into_the_pixel(oracle, m):
    """GlobalSampler contract: the s-th index of pixel p, scaled by the resolution, lands in pixel p."""
    L = oracle.load()
    res = 1 << m
    seen = set()
    for py in range(res):
        for px in range(res):
            for s in range(4):
                idx = L.orc_sobol_interval_to_index(m, s, px, py)
                assert idx not in seen
                seen.add(idx)
                x = L.orc_sobol_sample_float(idx, 0, 0) * res
                y = L.orc_sobol_sample_float(idx, 1, 0) * res
                assert int(x) == px and int(y) == py


def test_radical_inverse_exact_rationals(oracle):
    L = oracle.load()
    primes = [2, 3, 5, 7, 11]
    for bi, b in enumerate(primes):
        for a in range(128):
            digits, x = [], a
            while x:
                digits.append(x % b)
                x //= b
            want = sum(Fraction(d, b ** (i + 1)) for i, d in enumerate(digits))
            got = L.orc_radical_inverse(bi, a)
            assert abs(got - float(want)) <= 4e-7 * max(float(want), 1e-9)


def test_sobol_golden_vectors(oracle):
    L = oracle.load()
    g = np.load(GOLD / "sobol_kat.npz")
    got = np.array([[L.orc_sobol_sample_float(int(a), int(d), 0) for d in g["dims"]] for a in g["idx"]], np.float32)
    assert np.array_equal(got.view(np.uint32), g["sobol"].view(np.uint32))
    for m, f, x, y, want in g["interval"]:
        assert L.orc_sobol_interval_to_index(int(m), int(f), int(x), int(y)) == int(want)
    rad = np.array([[L.orc_radical_inverse(b, i) for b in range(5)] for i in range(128)], np.float32)
    assert np.array_equal(rad.view(np.uint32), g["radical"].view(np.uint32))


def _bsdf(L, mat, ns, ng, ss, wo, wi, u, flags=31):
    fp = lambda a: np.ascontiguousarray(a, np.float32).ctypes.data_as(C.POINTER(C.c_float))
    out = np.zeros(12, np.float32)
    m = _abi.PbrtMaterial()
    m.kind = mat[0]
    for i, v in enumerate(mat[1]):
        m.params[i] = v
    keep = [np.ascontiguousarray(a, np.float32) for a in (ns, ng, ss, wo, wi, u)]
    rc = L.orc_bsdf(C.byref(m), *[k.ctypes.data_as(C.POINTER(C.c_float)) for k in keep], flags, fp(out))
    assert rc == 0
    return out


MATS = {
    "matte": (_abi.MAT_MATTE, [0.5, 0.6, 0.7, 0.0]),
    "oren": (_abi.MAT_MATTE, [0.5, 0.6, 0.7, 25.0]),
    "plastic": (_abi.MAT_PLASTIC, [0.4, 0.3, 0.2, 0.3, 0.3, 0.3, 0.2, 1.0]),
    "metal": (_abi.MAT_METAL, [0.2, 0.92, 1.1, 3.9, 2.45, 2.14, 0.1, 0.2, 1.0]),
    "substrate": (_abi.MAT_SUBSTRATE, [0.4, 0.3, 0.2, 0.1, 0.1, 0.1, 0.1, 0.15, 1.0]),
    "uber": (_abi.MAT_UBER, [0.3, 0.3, 0.3, 0.2, 0.2, 0.2, 0, 0, 0, 0, 0, 0, 1, 1, 1, 0.1, 0.1, 1.5, 1.0]),
    "roughglass": (_abi.MAT_GLASS, [1, 1, 1, 1, 1, 1, 1.5, 0.2, 0.2, 1.0]),
    "translucent": (_abi.MAT_TRANSLUCENT, [0.6, 0.5, 0.3, 0.3, 0.3, 0.3, 0.5, 0.5, 0.5, 0.5, 0.5, 0.5, 0.15, 1.0]),
    "translucent_diffuse": (_abi.MAT_TRANSLUCENT, [0.6, 0.5, 0.3, 0.0, 0.0, 0.0, 0.4, 0.4, 0.4, 0.6, 0.6, 0.6, 0.15, 1.0]),
}
Z = [0.0, 0.0, 1.0]
X = [1.0, 0.0, 0.0]


@pytest.mark.parametrize("name", ["matte", "oren", "plastic", "metal", "substrate", "uber"])
def test_bsdf_reciprocity_and_sample_pdf_consistency(oracle, name):
    L = oracle.load()
    rng = np.random.default_rng(3)
    for _ in range(50):
        wo = rng.normal(size=3); wo[2] = abs(wo[2]) + 0.05; wo /= np.linalg.norm(wo)
        wi = rng.normal(size=3); wi[2] = abs(wi[2]) + 0.05; wi /= np.linalg.norm(wi)
        a = _bsdf(L, MATS[name], Z, Z, X, wo, wi, [0.3, 0.7], flags=31 & ~16)
        b = _bsdf(L, MATS[name], Z, Z, X, wi, wo, [0.3, 0.7], flags=31 & ~16)
        if name != "substrate":  # FresnelBlend's diffuse term is reciprocal, its specular term is not exactly
            assert np.allclose(a[:3], b[:3], rtol=2e-4, atol=1e-7)
        u = rng.uniform(0.01, 0.99, 2)
        s = _bsdf(L, MATS[name], Z, Z, X, wo, wi, u, flags=31 & ~16)
        f_s, pdf_s, wi_s = s[4:7], s[7], s[8:11]
        if pdf_s > 0:
            e = _bsdf(L, MATS[name], Z, Z, X, wo, wi_s, u, flags=31 & ~16)
            assert np.allclose(e[3], pdf_s, rtol=2e-3, atol=1e-6), (e[3], pdf_s)
            assert np.allclose(e[:3], f_s, rtol=2e-3, atol=1e-6)


@pytest.mark.parametrize("name", ["matte", "plastic", "metal", "substrate", "roughglass", "translucent", "translucent_diffuse"])
def test_bsdf_white_furnace_bounded(oracle, name):
    """The Monte-Carlo estimate of the albedo with the BSDF's own sampling equals the float64 quadrature albedo of
    tests/f64_reference.py within 5 standard errors (and a 1e-4 floor for the all-Lambert cases, whose estimate has no variance)."""
    import f64_reference

    L = oracle.load()
    rng = np.random.default_rng(5)
    wo = np.array([0.3, 0.2, 0.93]); wo /= np.linalg.norm(wo)
    n = 4000
    est = np.zeros((n, 3))
    for i in range(n):
        s = _bsdf(L, MATS[name], Z, Z, X, wo, wo, rng.uniform(0, 1, 2), flags=31)
        if s[7] > 0:
            est[i] = s[4:7] * abs(s[10]) / s[7]
    rho = f64_reference.albedo(f64_reference.material_lobes([MATS[name]], 0), wo, rtol=1e-5)
    se = est.std(0, ddof=1) / np.sqrt(n)
    assert np.all(np.abs(est.mean(0) - rho) <= 5 * se + 1e-4 * rho), (est.mean(0), rho, se)


def test_translucent_lobes(oracle):
    """TranslucentMaterial (translucent.rs:48-189) without Ks is LambertianReflection(reflect * Kd) + LambertianTransmission(transmit * Kd)
    (reflection.rs:1001-1046): the lobe is chosen by u[0], a transmitted direction lies in the other hemisphere with pdf |cos| / pi
    averaged over the two matching lobes, and f is the closed form on either side."""
    L = oracle.load()
    kind, p = MATS["translucent_diffuse"]
    kd, refl, tran = np.array(p[0:3]), np.array(p[6:9]), np.array(p[9:12])
    rng = np.random.default_rng(11)
    for _ in range(40):
        wo = rng.normal(size=3); wo[2] = abs(wo[2]) + 0.05; wo /= np.linalg.norm(wo)
        for ux, transmitted in ((rng.uniform(0.0, 0.49), False), (rng.uniform(0.51, 0.99), True)):
            s = _bsdf(L, (kind, p), Z, Z, X, wo, wo, [ux, rng.uniform(0.01, 0.99)], flags=31)
            f_s, pdf_s, wi_s = s[4:7], s[7], s[8:11]
            assert (wi_s[2] < 0) == transmitted
            want = (tran if transmitted else refl) * kd / np.pi
            assert np.allclose(f_s, want, rtol=1e-6)
            assert np.isclose(pdf_s, abs(wi_s[2]) / np.pi / 2.0, rtol=1e-5)  # the other lobe's pdf is 0 on this side
            e = _bsdf(L, (kind, p), Z, Z, X, wo, wi_s, [0.5, 0.5], flags=31)
            assert np.allclose(e[:3], want, rtol=1e-6) and np.isclose(e[3], pdf_s, rtol=1e-5)
    # black reflect and transmit: no lobes at all
    dead = list(p); dead[6:12] = [0.0] * 6
    s = _bsdf(L, (kind, dead), Z, Z, X, [0.0, 0.6, 0.8], [0.0, -0.6, 0.8], [0.3, 0.3], flags=31)
    assert np.all(s[:4] == 0) and s[7] == 0


def _bsdf_at(L, mats, index, ns, ng, ss, wo, wi, u, flags=31, want_rc=0):
    """Bsdf of material `index` of a material array ((kind, params) tuples; a MIX's params are amount[3], m1, m2)."""
    arr = (_abi.PbrtMaterial * len(mats))()
    for m, (kind, params) in zip(arr, mats):
        m.kind = kind
        for i, v in enumerate(params):
            m.params[i] = v
    out = np.zeros(12, np.float32)
    keep = [np.ascontiguousarray(a, np.float32) for a in (ns, ng, ss, wo, wi, u)]
    rc = L.orc_bsdf_at(arr, len(mats), index, *[k.ctypes.data_as(C.POINTER(C.c_float)) for k in keep], flags, out.ctypes.data_as(C.POINTER(C.c_float)))
    assert rc == want_rc
    return out


def test_mix_material_lobes(oracle):
    """MixMaterial (mixmat.rs:41-98): m1's BxDFs carry sc_opt = clamp(amount), m2's clamp(1 - that), both lists in one Bsdf.
    Two Lambertian lobes: f is the blend in closed form, the pdf the cosine pdf (averaged over two equal lobes).  An amount outside
    [0, 1] is clamped on both sides separately.  A lobe scaled to zero is still a lobe (it is counted among the matching components)."""
    L = oracle.load()
    kd1, kd2 = np.array([0.5, 0.6, 0.7], np.float32), np.array([0.2, 0.1, 0.4], np.float32)
    wo, wi = np.array([0.3, 0.2, 0.9327379], np.float32), np.array([-0.5, 0.1, 0.8602325], np.float32)
    for amount in ([0.25, 0.5, 1.0], [1.5, -0.5, 0.3]):
        a = np.array(amount, np.float32)
        s1 = np.clip(a, 0.0, None)
        s2 = np.clip(np.float32(1.0) - s1, 0.0, None)
        mats = [(_abi.MAT_MATTE, list(kd1) + [0.0]), (_abi.MAT_MATTE, list(kd2) + [0.0]), (_abi.MAT_MIX, amount + [0.0, 1.0])]
        e = _bsdf_at(L, mats, 2, Z, Z, X, wo, wi, [0.5, 0.5])
        inv_pi = np.float32(1.0 / np.pi)
        want = (s1 * kd1) * inv_pi + (s2 * kd2) * inv_pi  # (sc * r) * INV_PI per lobe, summed in lobe order (reflection.rs:963-965, :283-296)
        assert np.array_equal(e[:3], want.astype(np.float32))
        assert np.isclose(e[3], wi[2] / np.pi, rtol=1e-6)
        s = _bsdf_at(L, mats, 2, Z, Z, X, wo, wo, [0.7, 0.3])
        assert np.isclose(s[7], s[10] / np.pi, rtol=1e-6) and s[11] == (1 | 4)  # BSDF_REFLECTION | BSDF_DIFFUSE


def test_mix_material_specular_child_and_nested_mix(oracle):
    """A specular lobe's sc_opt acts in sample_f (reflection.rs:739-744): with Lambert + mirror under amount a, the second half of u[0]
    picks the mirror, f = (1 - a) * Kr / |cos|, pdf = 1 / 2.  A MixMaterial that is itself a child ignores the scale handed down
    (`_scale`, mixmat.rs:48): its lobes keep their own scales, only the sibling is scaled by the outer amount."""
    L = oracle.load()
    kd, kr = [0.5, 0.6, 0.7], [0.9, 0.8, 0.7]
    mats = [(_abi.MAT_MATTE, kd + [0.0]), (_abi.MAT_MIRROR, kr), (_abi.MAT_MIX, [0.25, 0.25, 0.25, 0.0, 1.0])]
    wo = np.array([0.3, 0.2, 0.9327379], np.float32)
    s = _bsdf_at(L, mats, 2, Z, Z, X, wo, wo, [0.75, 0.3])
    assert np.allclose(s[8:11], [-wo[0], -wo[1], wo[2]]) and s[7] == 0.5 and s[11] == (1 | 16)
    assert np.array_equal(s[4:7], (np.float32(0.75) * np.float32(1.0)) * np.array(kr, np.float32) / np.float32(wo[2]))
    d = _bsdf_at(L, mats, 2, Z, Z, X, wo, wo, [0.25, 0.3])  # first half: the Lambert lobe, alone among the non-specular ones
    assert np.array_equal(d[4:7], (np.float32(0.25) * np.array(kd, np.float32)) * np.float32(1.0 / np.pi))
    # nested: outer = mix(inner, matte2, 0.5) with inner = mix(matte, mirror, 0.25)
    kd2 = [0.1, 0.2, 0.3]
    nested = mats + [(_abi.MAT_MATTE, kd2 + [0.0]), (_abi.MAT_MIX, [0.5, 0.5, 0.5, 2.0, 3.0])]
    wi = np.array([-0.5, 0.1, 0.8602325], np.float32)
    e = _bsdf_at(L, nested, 4, Z, Z, X, wo, wi, [0.5, 0.5])
    inv_pi = np.float32(1.0 / np.pi)
    want = (np.float32(0.25) * np.array(kd, np.float32)) * inv_pi + (np.float32(0.5) * np.array(kd2, np.float32)) * inv_pi
    assert np.array_equal(e[:3], want)
    # three lobes now: {Lambert, mirror, Lambert}; u[0] in the middle third picks the mirror with the INNER scale 0.75 only
    s = _bsdf_at(L, nested, 4, Z, Z, X, wo, wo, [0.5, 0.3])
    assert s[11] == (1 | 16) and np.isclose(s[7], 1.0 / 3.0, rtol=1e-6)
    assert np.array_equal(s[4:7], (np.float32(0.75) * np.float32(1.0)) * np.array(kr, np.float32) / np.float32(wo[2]))


def test_mix_material_limits(oracle):
    """Bsdf::add asserts on a ninth BxDF (reflection.rs:246-249); children come before the mix that names them."""
    L = oracle.load()
    uber = (_abi.MAT_UBER, [0.3, 0.3, 0.3, 0.2, 0.2, 0.2, 0.1, 0.1, 0.1, 0.2, 0.2, 0.2, 0.5, 0.5, 0.5, 0.1, 0.1, 1.5, 1.0])  # five lobes
    wo = [0.3, 0.2, 0.9327379]
    _bsdf_at(L, [uber, uber, (_abi.MAT_MIX, [0.5, 0.5, 0.5, 0.0, 1.0])], 2, Z, Z, X, wo, wo, [0.5, 0.5], want_rc=-1)  # 10 lobes
    ok = _bsdf_at(L, [uber, MATS["plastic"], (_abi.MAT_MIX, [0.5, 0.5, 0.5, 0.0, 1.0])], 2, Z, Z, X, wo, wo, [0.5, 0.5])  # 7 lobes: fine in the reference
    assert ok[7] > 0
    _bsdf_at(L, [(_abi.MAT_MIX, [0.5, 0.5, 0.5, 0.0, 1.0]), uber], 0, Z, Z, X, wo, wo, [0.5, 0.5], want_rc=-1)  # names itself / a later material


@pytest.mark.parametrize("pair", [("matte", "oren"), ("plastic", "roughglass"), ("translucent", "oren"), ("substrate", "metal")])
def test_mix_white_furnace_bounded(oracle, pair):
    """A blend of two energy-conserving BSDFs with weights a and 1 - a conserves energy."""
    L = oracle.load()
    mats = [MATS[pair[0]], MATS[pair[1]], (_abi.MAT_MIX, [0.3, 0.5, 0.8, 0.0, 1.0])]
    rng = np.random.default_rng(4)
    wo = np.array([0.3, -0.2, 0.93], np.float32); wo /= np.linalg.norm(wo)
    acc, n = np.zeros(3), 3000
    for _ in range(n):
        s = _bsdf_at(L, mats, 2, Z, Z, X, wo, wo, rng.random(2))
        if s[7] > 0:
            acc += s[4:7] * abs(s[10]) / s[7]
    assert np.all(acc / n < 1.05), acc / n


def test_light_distribution_properties(oracle):
    h = scenes.cornell_box(xres=16, yres=16, spp=1)
    osc = oracle.OracleScene(h.desc)
    for strat in (0, 1, 2):
        func, cdf, fint = osc.light_distribution(strat, [100.0, 200.0, 300.0], 2)
        assert cdf[0] == 0.0 and abs(cdf[-1] - 1.0) < 1e-6 and np.all(np.diff(cdf) >= 0)
        assert np.all(func > 0) and fint > 0
    # near the light the spatial distribution prefers the nearer light triangle; uniform stays uniform
    f_uni, _, _ = osc.light_distribution(0, [300.0, 500.0, 240.0], 2)
    assert f_uni[0] == f_uni[1]


def test_film_add_sample_footprint(oracle):
    """film.rs:94-147: box filter radius 0.5 hits the sample's own pixel; an offset of exactly 0 also hits x-1."""
    L = oracle.load()
    h = scenes.cornell_box(xres=8, yres=8, spp=1)
    rp = h.params
    fp = lambda a: a.ctypes.data_as(C.POINTER(C.c_float))
    film = np.zeros((8, 8, 4), np.float32)
    L.orc_film_add_sample(rp, fp(film), fp(np.array([3.25, 4.75], np.float32)), fp(np.array([1, 2, 3], np.float32)), 1.0)
    assert film[4, 3].tolist() == [1, 2, 3, 1] and film.sum() == 7
    film[:] = 0
    L.orc_film_add_sample(rp, fp(film), fp(np.array([3.0, 4.5], np.float32)), fp(np.array([1, 1, 1], np.float32)), 1.0)
    assert film[4, 3, 3] == 1 and film[4, 2, 3] == 1 and film[..., 3].sum() == 2
    film[:] = 0
    L.orc_film_add_sample(rp, fp(film), fp(np.array([0.0, 0.0], np.float32)), fp(np.array([1, 1, 1], np.float32)), 1.0)
    assert film[..., 3].sum() == 1  # neighbours outside the cropped bounds are dropped


def test_cornell_golden_fixture(oracle):
    g = np.load(GOLD / "cornell_32x32x8.npz")
    h = scenes.cornell_box(xres=32, yres=32, spp=8)
    osc = oracle.OracleScene(h.desc)
    prim, t, b, st = osc.intersect(g["o"], g["d"])
    assert np.array_equal(prim, g["prim"]) and np.array_equal(t.view(np.uint32), g["t"].view(np.uint32))
    assert np.array_equal(b.view(np.uint32), g["b"].view(np.uint32))
    assert st["nodes_visited"] == int(g["nodes_visited"]) and st["tris_tested"] == int(g["tris_tested"])
    occ, _ = osc.intersect_p(g["o"], g["d"] * np.float32(250.0), np.full(len(g["o"]), 1.0 - 1e-4, np.float32))
    assert np.array_equal(occ, g["occ"])
    cam = np.array([osc.camera_sample(h.params, px, py, s) for (px, py, s) in ((0, 0, 0), (5, 7, 3), (31, 31, 7), (16, 2, 5))], np.float32)
    assert np.array_equal(cam.view(np.uint32), g["cam"].view(np.uint32))
    film, samples, rst = osc.render(h.params, n_threads=2, want_samples=True)
    assert rst["rays"] == int(g["rays"])
    # radiance goes through libm sinf/cosf whose last bit may differ between CPU variants
    assert np.allclose(samples, g["samples"], rtol=1e-5, atol=1e-7)
    assert np.allclose(film, g["film"], rtol=1e-5, atol=1e-6)
    for i, p in enumerate(g["ld_pts"]):
        func, cdf, fint = osc.light_distribution(2, p, 2)
        assert np.array_equal(func, g["ld_func"][i]) and np.array_equal(cdf, g["ld_cdf"][i]) and fint == g["ld_int"][i]


def test_mixed_materials_golden_fixture(oracle):
    g = np.load(GOLD / "cornell_mixed_24x24x8.npz")
    h = scenes.cornell_box(xres=24, yres=24, spp=8, materials="mixed")
    film, samples, rst = oracle.OracleScene(h.desc).render(h.params, n_threads=2, want_samples=True)
    assert abs(rst["rays"] - int(g["rays"])) <= 2
    bad = ~np.isclose(samples, g["samples"], rtol=1e-4, atol=1e-6).all(axis=-1)
    assert bad.mean() < 1e-3
    assert np.all(np.isfinite(film))


def test_render_is_thread_count_invariant(oracle):
    h = scenes.cornell_box(xres=24, yres=24, spp=4)
    osc = oracle.OracleScene(h.desc)
    f1, s1, _ = osc.render(h.params, n_threads=1, want_samples=True)
    f8, s8, _ = osc.render(h.params, n_threads=8, want_samples=True)
    assert np.array_equal(s1, s8)
    assert np.allclose(f1, f8, rtol=1e-6)


def test_widened_golden_fixture(oracle):
    """tests/golden/widened_16.npz: textures + bump maps, object instances in both instancing modes, direct / whitted / ao -- the oracle
    still answers what it answered when the fixture was frozen."""
    from golden_cases import widened_cases
    g = np.load(GOLD / "widened_16.npz")
    for name, h in widened_cases():
        _, samples, st = oracle.OracleScene(h.desc).render(h.params, n_threads=2, want_samples=True)
        assert st["rays"] == int(g[name + "_rays"]), name
        assert np.array_equal(samples, g[name + "_samples"]), name


def test_round2_golden_fixture(oracle):
    """tests/golden/round2_16.npz: alpha masks, TranslucentMaterial, MixMaterial under path / whitted / directlighting with Halton -- frozen like the others."""
    from golden_cases import round2_cases
    g = np.load(GOLD / "round2_16.npz")
    for name, h in round2_cases():
        _, samples, st = oracle.OracleScene(h.desc).render(h.params, n_threads=2, want_samples=True)
        assert st["rays"] == int(g[name + "_rays"]), name
        assert np.array_equal(samples, g[name + "_samples"]), name
