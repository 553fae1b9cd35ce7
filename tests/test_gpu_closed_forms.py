"""The CUDA path integrator against float64 closed forms (tests/f64_reference.py), not against the oracle.  Every scene is built
with HostScene and rendered per sample with GpuScene.render_samples.  The oracle is used for one thing only: the f32 camera ray of
a sample (OracleScene.camera_sample), which the parity tests hold bit-identical to the GPU's.  Hit points, directions and expected
values are float64, computed from that ray.

A  BSDF values under delta lights, per sample: maxdepth = 1 and one point (or distant) light make every sample's radiance exactly
   f(wo, wi) I |cos th_i| / d^2.  Path and direct-lighting integrators alike.
B  specular outcomes under a constant sky, per sample, and the share of reflected glass samples against F(cos th_o).
C  unbiasedness: area lights over a Lambertian floor against Lambert's polygon formula (C1), glossy and transmissive floors under
   a constant sky against the quadrature albedo (C2), and a furnace for the multi-bounce throughput and Russian roulette (C3).
   With Halton and samplepixelcenter every sample of a pixel shares one hit point and one expectation; the aggregate relative bias
   is held to 5 sample standard errors and the largest per-pixel |z| to a Bonferroni bound.  Every case also asserts that its
   standard error is at most 0.25 % of the expectation, so that a 2 % bias is at least 8 standard errors and fails."""
import math

import numpy as np
import pytest
from scipy import stats

import f64_reference as R
from rs_pbrt_b200 import GpuScene, HostScene

pytestmark = pytest.mark.gpu

FLOOR = np.array([[-60, 0, -60], [60, 0, -60], [60, 0, 60], [-60, 0, 60]], np.float32)
FLOOR_IDX = [0, 2, 1, 0, 3, 2]  # both triangles face +y
FLOOR_UV = np.array([[0, 0], [1, 0], [1, 1], [0, 1]], np.float32)  # u grows along +x: dpdu, hence the shading tangent, is +x
UP = np.array([0.0, 1.0, 0.0])
SS = np.array([1.0, 0.0, 0.0])


def render(h):
    g = GpuScene(h.desc, 0)
    try:
        s, st = g.render_samples(h.params, list(h.params.contents.sample_bounds))
    finally:
        g.close()
    assert np.all(np.isfinite(s))
    return s.astype(np.float64), st


def camera_rays(h, oracle):
    """(H, W, spp, 3) origins and directions of the camera samples, float64 copies of the f32 rays."""
    rp = h.params.contents
    sb = list(rp.sample_bounds)
    orc = oracle.OracleScene(h.desc)
    o = np.zeros((sb[3] - sb[1], sb[2] - sb[0], rp.spp, 3))
    d = np.zeros_like(o)
    for y in range(sb[1], sb[3]):
        for x in range(sb[0], sb[2]):
            for s in range(rp.spp):
                c = orc.camera_sample(h.params, x, y, s).astype(np.float64)
                o[y - sb[1], x - sb[0], s], d[y - sb[1], x - sb[0], s] = c[5:8], c[8:11]
    orc.close()
    return o, d


def floor_hits(o, d):
    t = -o[..., 1] / d[..., 1]
    assert np.all(t > 0)
    p = o + d * t[..., None]
    assert np.all(np.abs(p[..., 0]) < 60) and np.all(np.abs(p[..., 2]) < 60)
    return p


def scene(mats, floor_mat, lights, spp=4, res=24, integrator=("path", 1), sampler="sobol", center=False, eye=(0, 5, -5), look=(0, 0, 0.5), fov=50.0):
    """mats: (kind, params) list in creation order (a MIX names earlier entries); the floor gets material `floor_mat`.
    lights(h) declares the lights and any emitters."""
    h = HostScene()
    for kind, p in mats:
        if kind == R.MIX:
            h.material_mix(int(p[3]), int(p[4]), p[0:3])
        else:
            h.material(kind, p)
    h.trianglemesh(FLOOR_IDX, FLOOR, UV=FLOOR_UV, material=floor_mat)
    lights(h)
    h.look_at(list(eye), list(look), [0, 1, 0])
    h.film(res, res)
    h.camera(fov=fov)
    h.sampler(spp, name=sampler, samplepixelcenter=center)
    if integrator[0] == "path":
        h.integrator(maxdepth=integrator[1], rrthreshold=integrator[2] if len(integrator) > 2 else 1.0,
                     lightsamplestrategy=integrator[3] if len(integrator) > 3 else "spatial")
    else:
        h.integrator_direct(maxdepth=integrator[1], strategy="all")
    h.world_end()
    return h


# ---- A: BSDF values under delta lights ------------------------------------------------------------------------------------

MATERIALS = {
    "matte": [(R.MATTE, [0.5, 0.6, 0.7, 0.0])],
    "matte-sigma20": [(R.MATTE, [0.5, 0.6, 0.7, 20.0])],
    "plastic-rough0.1-remap": [(R.PLASTIC, [0.3, 0.2, 0.1, 0.6, 0.5, 0.4, 0.1, 1.0])],
    "plastic-rough0.05-noremap": [(R.PLASTIC, [0.3, 0.2, 0.1, 0.6, 0.5, 0.4, 0.05, 0.0])],
    "plastic-rough0.4-noremap": [(R.PLASTIC, [0.3, 0.2, 0.1, 0.6, 0.5, 0.4, 0.4, 0.0])],
    "metal-iso-remap": [(R.METAL, [0.2, 0.92, 1.1, 3.9, 2.45, 2.14, 0.1, 0.1, 1.0])],
    "metal-iso-noremap": [(R.METAL, [0.2, 0.92, 1.1, 3.9, 2.45, 2.14, 0.2, 0.2, 0.0])],
    "metal-aniso-remap": [(R.METAL, [1.66, 0.88, 0.52, 9.2, 6.27, 4.84, 0.05, 0.3, 1.0])],
    "metal-aniso-noremap": [(R.METAL, [1.66, 0.88, 0.52, 9.2, 6.27, 4.84, 0.1, 0.35, 0.0])],
    "substrate-iso": [(R.SUBSTRATE, [0.4, 0.3, 0.2, 0.08, 0.06, 0.04, 0.15, 0.15, 0.0])],
    "substrate-aniso": [(R.SUBSTRATE, [0.4, 0.3, 0.2, 0.08, 0.06, 0.04, 0.05, 0.3, 0.0])],
    "uber-opaque": [(R.UBER, [0.3, 0.25, 0.2, 0.4, 0.4, 0.4, 0, 0, 0, 0, 0, 0, 1, 1, 1, 0.12, 0.2, 1.6, 0.0])],
    "uber-opacity0.6": [(R.UBER, [0.3, 0.25, 0.2, 0.4, 0.4, 0.4, 0, 0, 0, 0, 0, 0, 0.6, 0.7, 0.8, 0.12, 0.2, 1.6, 0.0])],
    "roughglass": [(R.GLASS, [0.9, 0.9, 0.9, 0.8, 0.9, 1.0, 1.5, 0.15, 0.3, 0.0])],
    "translucent": [(R.TRANSLUCENT, [0.6, 0.5, 0.3, 0.3, 0.3, 0.3, 0.5, 0.6, 0.7, 0.5, 0.4, 0.3, 0.2, 0.0])],
    "mix-plastic-metal": [(R.PLASTIC, [0.3, 0.2, 0.1, 0.6, 0.5, 0.4, 0.1, 1.0]), (R.METAL, [1.66, 0.88, 0.52, 9.2, 6.27, 4.84, 0.1, 0.35, 0.0]),
                          (R.MIX, [0.3, 0.5, 0.8, 0, 1])],
    "mirror": [(R.MIRROR, [0.9, 0.8, 0.7])],
    "smoothglass": [(R.GLASS, [0.9, 0.9, 0.9, 0.8, 0.9, 1.0, 1.5, 0.0, 0.0, 0.0])],
}
TRANSMISSIVE = ("roughglass", "translucent")
POINT = (np.array([1.5, 3.0, 2.0]), np.array([20.0, 15.0, 10.0]))
POINT_BELOW = (np.array([-0.5, -2.5, 1.5]), np.array([20.0, 15.0, 10.0]))
DISTANT = (np.array([1.0, 2.0, -0.5]), np.array([3.0, 2.0, 1.0]))

CASES = [(m, "point") for m in MATERIALS] + [(m, "distant") for m in MATERIALS if m not in ("mirror", "smoothglass")] + \
        [(m, "point-below") for m in TRANSMISSIVE]


def delta_expectation(mats, floor_mat, light, o, d):
    """f(wo, wi) L |cos th_i| (/ d^2 for a point light) at every sample's floor hit."""
    p = floor_hits(o, d)
    wo = -d / np.linalg.norm(d, axis=-1, keepdims=True)
    kind, pos, I = light
    if kind == "distant":
        wi = np.broadcast_to(pos / np.linalg.norm(pos), p.shape)
        li = np.broadcast_to(I, p.shape)
    else:
        v = pos - p
        d2 = np.sum(v * v, -1, keepdims=True)
        wi = v / np.sqrt(d2)
        li = I / d2
    lobes = R.material_lobes(mats, floor_mat)
    f = R.bsdf_f_world(lobes, UP, SS, UP, wo, wi)
    # Error estimate: the kernel sees wo and wi as f32 vectors, a few ulps (~1e-7) off the float64 ones.  Moving either by DIR_ERR
    # along the tangent axes bounds what that does to f.  It is ~1e-6 relative everywhere except at the critical angle of a dielectric
    # Fresnel term (plastic's 1.5 -> 1 interface), where cos th_t = sqrt(1 - sin^2 th_t) turns a 1e-7 change of the angle into ~1e-4.
    sens = np.zeros(f.shape)
    for axis in (np.array([DIR_ERR, 0, 0]), np.array([0, 0, DIR_ERR])):
        for sign in (1, -1):
            for a, b in ((wo + sign * axis, wi), (wo, wi + sign * axis)):
                fp = R.bsdf_f_world(lobes, UP, SS, UP, R._normalize(a), R._normalize(b))
                sens = np.maximum(sens, np.abs(fp - f))
    return f * li * np.abs(wi[..., 1:2]), np.abs(wi[..., 1]), sens * li * np.abs(wi[..., 1:2])


DIR_ERR = 1e-6  # ten f32 ulps of a unit vector's component


@pytest.mark.parametrize("integrator", [("path", 1), ("direct", 1)], ids=["path", "direct"])
@pytest.mark.parametrize("name,light", CASES, ids=["%s-%s" % c for c in CASES])
def test_bsdf_value_under_delta_light(oracle, name, light, integrator):
    mats = MATERIALS[name]
    lt = {"point": ("point",) + POINT, "point-below": ("point",) + POINT_BELOW, "distant": ("distant",) + DISTANT}[light]

    def lights(h):
        if lt[0] == "point":
            h.light_point(lt[1], lt[2])
        else:
            h.light_distant(lt[1], [0, 0, 0], lt[2])

    h = scene(mats, len(mats) - 1, lights, integrator=integrator)
    got, _ = render(h)
    o, d = camera_rays(h, oracle)
    want, cos_i, sens = delta_expectation(mats, len(mats) - 1, lt, o, d)
    if name in ("mirror", "smoothglass"):
        assert np.all(got == 0.0)
        return
    assert np.all(cos_i > 1e-2)  # no grazing light in these scenes
    scale = float(np.max(want))
    assert scale > 0 and np.count_nonzero(want) > 0.1 * want.size  # (a narrow transmission lobe lights only part of the floor)
    denom = np.maximum(np.abs(want), 1e-3 * scale)
    err = np.abs(got - want) / denom
    loose = sens / denom > 1e-4  # where the direction error estimate alone exceeds the 1e-4 bound
    print("%s %s %s: worst relative error %.2e; %d samples near a critical angle, worst %.2e against their own bound"
          % (name, light, integrator[0], float(err[~loose].max()), int(loose.sum()), float((err / (1e-4 + sens / denom))[loose].max(initial=0))))
    assert float(err[~loose].max()) <= 1e-4
    assert np.all(err <= 1e-4 + sens / denom)
    assert np.count_nonzero(loose) <= 0.01 * loose.size


# ---- B: specular outcomes under a constant sky ------------------------------------------------------------------------------

LS = np.array([0.7, 0.8, 0.9])


def sky(h):
    h.light_infinite(LS)


def test_mirror_reflects_the_sky(oracle):
    kr = np.array([0.9, 0.8, 0.7])
    h = scene([(R.MIRROR, list(kr))], 0, sky)
    got, _ = render(h)
    assert np.allclose(got, kr * LS, rtol=1e-6, atol=0)


def test_smooth_glass_reflects_or_transmits_with_fresnel_odds(oracle):
    kr, kt, eta = np.array([0.9, 0.8, 0.7]), np.array([0.5, 0.7, 0.9]), 1.5
    h = scene([(R.GLASS, list(kr) + list(kt) + [eta, 0.0, 0.0, 0.0])], 0, sky, spp=16, res=32)
    got, _ = render(h)
    refl, tran = kr * LS, kt * LS / eta ** 2
    is_r = np.all(np.isclose(got, refl, rtol=1e-6, atol=0), -1)
    is_t = np.all(np.isclose(got, tran, rtol=1e-6, atol=0), -1)
    assert np.all(is_r | is_t)
    o, d = camera_rays(h, oracle)
    F = R.fr_dielectric(-d[..., 1] / np.linalg.norm(d, axis=-1), 1.0, eta)
    n_r, e_r = int(is_r.sum()), float(F.sum())
    sd = math.sqrt(float(np.sum(F * (1 - F))))
    print("reflected %d of %d, expected %.1f +- %.1f" % (n_r, F.size, e_r, sd))
    assert abs(n_r - e_r) <= 5 * sd


# ---- C: unbiasedness -------------------------------------------------------------------------------------------------------

def check_unbiased(got, want, mask, label, max_rel_se=2.5e-3, alpha=1e-3):
    """got (H, W, S, 3) samples, want (H, W, 3) expectations of the pixels where mask is set."""
    x, e = got[mask], want[mask]  # (P, S, 3), (P, 3)
    S = x.shape[1]
    ch = np.sum(e, 0) > 0
    tot, etot = np.sum(x, (0, 1)), S * np.sum(e, 0)
    se = np.sqrt(S * np.sum(np.var(x, axis=1, ddof=1), 0))
    rel_bias, rel_se = (tot - etot)[ch] / etot[ch], se[ch] / etot[ch]
    zpix = (np.mean(x, 1) - e) / np.maximum(np.std(x, axis=1, ddof=1) / math.sqrt(S), 1e-12 * np.maximum(e, 1e-30))
    zmax = stats.norm.isf(alpha / (2 * zpix.size))
    print("%s: relative bias %s, relative SE %s, max |z| %.2f (bound %.2f, %d pixels)" % (label, np.round(rel_bias, 5), np.round(rel_se, 5),
                                                                                      float(np.max(np.abs(zpix))), zmax, x.shape[0]))
    assert np.all(rel_se <= max_rel_se), "too few samples to detect a 2 %% bias: relative SE %s" % rel_se
    assert np.all(np.abs(rel_bias) <= 5 * rel_se), (rel_bias, rel_se)
    assert float(np.max(np.abs(zpix))) <= zmax


def quad(center, ex, ey):
    c, ex, ey = (np.asarray(v, np.float64) for v in (center, ex, ey))
    return np.array([c - ex - ey, c + ex - ey, c + ex + ey, c - ex + ey])


def emitter_normal(v):
    return R._normalize(np.cross(v[0] - v[2], v[1] - v[2]))


def ray_hits_polygon(o, d, v):
    """(...) bool: the rays o + t d, t > 0 cross the planar convex polygon v (m, 3)."""
    n = np.cross(v[1] - v[0], v[2] - v[0])
    t = np.sum((v[0] - o) * n, -1) / np.sum(d * n, -1)
    q = o + d * t[..., None]
    inside = np.ones(t.shape, bool)
    for i in range(len(v)):
        inside &= np.sum(np.cross(v[(i + 1) % len(v)] - v[i], q - v[i]) * n, -1) >= 0
    return inside & (t > 0)


KD = np.array([0.6, 0.5, 0.4])
EMITTERS = {  # (vertices in the order the mesh is given, Le, two_sided); the horizontal ones share one height, so none shades another
    "one": [(quad([0.3, 2.0, 1.0], [0.8, 0.0, 0.0], [0.0, 0.0, 0.6]), [6.0, 5.0, 4.0], False)],
    "three": [(quad([-1.5, 2.0, 1.5], [0.3, 0.0, 0.0], [0.0, 0.0, 0.3]), [40.0, 30.0, 20.0], False),
              (quad([1.2, 2.0, 0.5], [0.5, 0.0, 0.0], [0.0, 0.0, 0.7]), [5.0, 6.0, 7.0], False),
              (quad([0.0, 2.0, 3.0], [1.5, 0.0, 0.0], [0.0, 0.0, 1.0]), [1.0, 1.5, 2.0], False)],
    "two-sided-back": [(quad([0.3, 2.0, 1.0], [0.0, 0.0, 0.6], [0.8, 0.0, 0.0]), [6.0, 5.0, 4.0], True)],
    "horizon": [(quad([0.0, 0.5, 2.0], [0.0, 1.5, 0.0], [1.5, 0.0, 0.0]), [3.0, 4.0, 5.0], False)],  # crosses y = 0, faces -z
}


def area_scene(name, strategy, spp, res=16):
    def lights(h):
        m = h.material(R.MATTE, [0.5, 0.5, 0.5, 0.0])
        for v, le, two in EMITTERS[name]:
            h.trianglemesh([0, 1, 2, 0, 2, 3], v.astype(np.float32), material=m, emit=le, two_sided=two)
    return scene([(R.MATTE, list(KD) + [0.0])], 0, lights, spp=spp, res=res, sampler="halton", center=True, integrator=("path", 1, 1.0, strategy))


@pytest.mark.parametrize("name,strategy,spp", [("one", "spatial", 1024), ("three", "uniform", 2048), ("three", "power", 2048), ("three", "spatial", 2048),
                                               ("two-sided-back", "spatial", 1024), ("horizon", "power", 4096)])
def test_area_lights_on_lambertian_floor(oracle, name, strategy, spp):
    h = area_scene(name, strategy, spp)
    got, _ = render(h)
    o, d = camera_rays(h, oracle)
    o, d = o[:, :, 0], d[:, :, 0]  # samplepixelcenter: one ray per pixel
    mask = np.ones(o.shape[:2], bool)
    for v, _, _ in EMITTERS[name]:
        mask &= ~ray_hits_polygon(o, d, v)  # pixels that see an emitter are not floor pixels
    p = floor_hits(o, d)
    want = np.zeros(p.shape)
    for y in range(p.shape[0]):
        for x in range(p.shape[1]):
            for v, le, two in EMITTERS[name]:
                if two or np.dot(emitter_normal(v), p[y, x] - v[0]) > 0:  # one-sided emitters light the side their normal is on
                    want[y, x] += KD / math.pi * np.asarray(le) * R.polygon_form_factor(p[y, x], UP, v)
    for v, _, two in EMITTERS[name]:  # every emitter faces the floor, but for the one seen from its back
        assert np.dot(emitter_normal(v), UP) < -0.99 or (two and np.dot(emitter_normal(v), UP) > 0.99) or name == "horizon"
    if name == "horizon":
        assert np.dot(emitter_normal(EMITTERS[name][0][0]), [0, 0, -1]) > 0.99
        assert np.any(want[mask][:, 0] == 0) and np.any(want[mask][:, 0] > 0)  # pixels behind the emitter and in front of it
    else:
        assert np.all(want[mask] > 0)
    check_unbiased(got, want, mask, "%s/%s" % (name, strategy))


GLOSSY = {
    "plastic": [(R.PLASTIC, [0.3, 0.2, 0.1, 0.6, 0.5, 0.4, 0.1, 1.0])],
    "metal-iso-narrow": [(R.METAL, [0.2, 0.92, 1.1, 3.9, 2.45, 2.14, 0.1, 0.1, 0.0])],
    "metal-aniso": [(R.METAL, [1.66, 0.88, 0.52, 9.2, 6.27, 4.84, 0.1, 0.35, 0.0])],
    "substrate-aniso": [(R.SUBSTRATE, [0.4, 0.3, 0.2, 0.08, 0.06, 0.04, 0.1, 0.3, 0.0])],
    "roughglass": [(R.GLASS, [0.9, 0.9, 0.9, 0.8, 0.9, 1.0, 1.5, 0.15, 0.3, 0.0])],
    "translucent": [(R.TRANSLUCENT, [0.6, 0.5, 0.3, 0.3, 0.3, 0.3, 0.5, 0.6, 0.7, 0.5, 0.4, 0.3, 0.2, 0.0])],
    "oren-nayar": [(R.MATTE, [0.5, 0.6, 0.7, 30.0])],
    "mix-substrate-glass": [(R.SUBSTRATE, [0.4, 0.3, 0.2, 0.08, 0.06, 0.04, 0.1, 0.3, 0.0]), (R.GLASS, [0.9, 0.9, 0.9, 0.8, 0.9, 1.0, 1.5, 0.15, 0.3, 0.0]),
                            (R.MIX, [0.4, 0.5, 0.6, 0, 1])],
}


# The quadrature of a microfacet transmission lobe converges to ~5e-6 at these resolutions (the critical-angle edge of F(wo . wh) is
# a curve across the grid); 1e-5 is still 100 times below the standard error of the estimate it is compared with.
RHO_RTOL = 1e-5


@pytest.mark.parametrize("name", list(GLOSSY))
def test_glossy_floor_under_constant_sky(oracle, name):
    """E[L] = Ls rho(wo): the density sample_f draws must be the pdf() it reports, or the MIS-weighted BSDF samples are biased."""
    mats = GLOSSY[name]
    h = scene(mats, len(mats) - 1, sky, spp=262144, res=1, sampler="halton", center=True, eye=(0, 3, -4), look=(0, 0, 0), fov=30.0)
    got, _ = render(h)
    o, d = camera_rays(h, oracle)
    d = d[:, :, 0] / np.linalg.norm(d[:, :, 0], axis=-1, keepdims=True)
    lobes = R.material_lobes(mats, len(mats) - 1)
    want = np.zeros(d.shape)
    for y in range(d.shape[0]):
        for x in range(d.shape[1]):
            wo = -d[y, x]
            want[y, x] = LS * R.albedo(lobes, np.array([wo @ SS, wo @ np.cross(UP, SS), wo @ UP]), panels=64, n_phi=1024, rtol=RHO_RTOL)
    check_unbiased(got, want, np.ones(d.shape[:2], bool), name)


def furnace(a, le, maxdepth, integrator="path", spp=512, res=16):
    h = HostScene()
    m = h.material(R.MATTE, list(a) + [0.0])
    corners = np.array([[x, y, z] for x in (-1, 1) for y in (-1, 1) for z in (-1, 1)], np.float64)
    faces = [(0, 1, 3, 2), (4, 6, 7, 5), (0, 4, 5, 1), (2, 3, 7, 6), (0, 2, 6, 4), (1, 5, 7, 3)]
    for f in faces:
        v = corners[list(f)]
        idx = [0, 1, 2, 0, 2, 3]
        if np.dot(emitter_normal(v), v.mean(0)) > 0:  # make every triangle face the inside
            idx = [0, 2, 1, 0, 3, 2]
        h.trianglemesh(idx, v.astype(np.float32), material=m, emit=list(le))
    h.look_at([0.1, -0.2, 0.05], [0.7, 0.3, 0.9], [0, 1, 0])
    h.film(res, res)
    h.camera(fov=70.0)
    h.sampler(spp)
    if integrator == "path":
        h.integrator(maxdepth=maxdepth, rrthreshold=1.0, lightsamplestrategy="spatial")
    else:
        h.integrator_direct(maxdepth=maxdepth, strategy="all")
    h.world_end()
    return h


@pytest.mark.parametrize("integrator,maxdepth", [("path", 1), ("path", 6), ("direct", 5)])
def test_furnace(integrator, maxdepth):
    """A closed cube of inward-facing emitters Le with albedo a: E[L] = Le sum_{k <= maxdepth} a^k for the path integrator (Russian
    roulette from the fourth bounce on at maxdepth 6), Le (1 + a) for direct lighting."""
    a, le = np.array([0.3, 0.5, 0.7]), np.array([1.0, 2.0, 0.5])
    h = furnace(a, le, maxdepth, integrator)
    got, _ = render(h)
    k = maxdepth if integrator == "path" else 1
    want = le * sum(a ** i for i in range(k + 1))
    W = np.broadcast_to(want, got.shape[:2] + (3,))
    check_unbiased(got, W, np.ones(got.shape[:2], bool), "furnace %s maxdepth %d" % (integrator, maxdepth))
