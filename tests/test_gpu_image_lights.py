"""Goniometric and projection lights (GonioPhotometricLight, ProjectionLight) on the CUDA path, against float64 closed forms.

At maxdepth 1 a matte floor lit by one delta light gives, per sample, Kd/pi * I * S(w) * |cos th| / d^2, where S is the light's image
lookup toward the shading point.  S is computed here in float64, independently of the library: the goniometric angles (world_to_light,
normalised, y and z swapped, theta / pi down the rows and phi / 2pi across) or the perspective projection onto the screen window of the
projection light, then a bilinear level-0 lookup with Repeat wrap.  As in test_gpu_closed_forms.py the oracle supplies only the f32
camera ray of each sample (it has no image lights, so it is handed the same scene with point lights in their place).
A goniometric light without a map must equal a point light bit for bit."""
import ctypes as C

import numpy as np
import pytest

from rs_pbrt_b200 import GpuScene, HostScene, _abi, scenes

pytestmark = pytest.mark.gpu

FLOOR = np.array([[-6, 0, -6], [6, 0, -6], [6, 0, 6], [-6, 0, 6]], np.float32)
FLOOR_IDX = [0, 2, 1, 0, 3, 2]
KD = np.array([0.5, 0.6, 0.7])
I = np.array([20.0, 15.0, 10.0])
POS = np.array([0.4, 2.5, 0.9])


ROT_Y90 = np.array([[0, 0, 1, 0], [0, 1, 0, 0], [-1, 0, 0, 0], [0, 0, 0, 1]], np.float64)  # maps the floor square onto itself


def floor_scene(lights, spp=2, res=32, integrator="path", strategy="spatial", sampler="sobol", instanced=False):
    """integrator: "path" | "direct" (= ("direct", "all")) | ("direct", "one") | "whitted", all at maxdepth 1.  instanced: the floor is an
    object instance turned 90 degrees about y (instancing "fixed"), which runs the instanced k_shade instantiations."""
    h = HostScene()
    h.material(_abi.MAT_MATTE, list(KD) + [0.0])
    if instanced:
        h.instancing("fixed")
        obj = h.object_begin()
        h.trianglemesh(FLOOR_IDX, FLOOR, material=0)
        h.object_end()
        h.object_instance(obj, ROT_Y90)
    else:
        h.trianglemesh(FLOOR_IDX, FLOOR, material=0)
    lights(h)
    h.look_at([0, 5, -5], [0, 0, 0.5], [0, 1, 0])
    h.film(res, res)
    h.camera(fov=60.0)
    h.sampler(spp, name=sampler)
    if integrator == "path":
        h.integrator(maxdepth=1, lightsamplestrategy=strategy)
    elif integrator == "whitted":
        h.integrator_whitted(maxdepth=1)
    else:
        h.integrator_direct(maxdepth=1, strategy="all" if integrator == "direct" else integrator[1])
    h.world_end()
    return h


def render(h):
    g = GpuScene(h.desc, 0)
    try:
        s, st = g.render_samples(h.params, list(h.params.contents.sample_bounds))
    finally:
        g.close()
    return s, st


def camera_rays(h, oracle):
    """float64 copies of the f32 camera rays, from the oracle given the scene with point lights in place of the image lights"""
    d = h.desc.contents
    kinds = [d.lights[i].kind for i in range(d.n_lights)]
    for i in range(d.n_lights):
        d.lights[i].kind = _abi.LIGHT_POINT
    try:
        rp = h.params.contents
        sb = list(rp.sample_bounds)
        orc = oracle.OracleScene(h.desc)
        o = np.zeros((sb[3] - sb[1], sb[2] - sb[0], rp.spp, 3))
        dd = np.zeros_like(o)
        for y in range(sb[1], sb[3]):
            for x in range(sb[0], sb[2]):
                for s in range(rp.spp):
                    c = orc.camera_sample(h.params, x, y, s).astype(np.float64)
                    o[y - sb[1], x - sb[0], s], dd[y - sb[1], x - sb[0], s] = c[5:8], c[8:11]
        orc.close()
    finally:
        for i, k in enumerate(kinds):
            d.lights[i].kind = k
    return o, dd


def bilinear(img, s, t):
    """MipMap::triangle(0, st) with Repeat wrap on a power-of-two (h, w, 3) map, in float64"""
    hh, ww = img.shape[:2]
    s = s * ww - 0.5
    t = t * hh - 0.5
    s0, t0 = np.floor(s).astype(np.int64), np.floor(t).astype(np.int64)
    ds, dt = (s - s0)[..., None], (t - t0)[..., None]
    tx = lambda a, b: img[b % hh, a % ww].astype(np.float64)
    return (1 - ds) * (1 - dt) * tx(s0, t0) + (1 - ds) * dt * tx(s0, t0 + 1) + ds * (1 - dt) * tx(s0 + 1, t0) + ds * dt * tx(s0 + 1, t0 + 1)


def turned(pos, ax, ay):
    return scenes.gonio_transform(pos, ax, ay)


def f32_inverse(m):
    return np.linalg.inv(m).astype(np.float32).astype(np.float64)


def expectation(o, d, S_of):
    """Kd/pi * I * S(-wi) * cos / d^2 at every floor hit; S_of(w_world) -> (S, keep)"""
    t = -o[..., 1] / d[..., 1]
    p = o + d * t[..., None]
    v = POS - p
    d2 = np.sum(v * v, -1, keepdims=True)
    wi = v / np.sqrt(d2)
    S, keep = S_of(-wi)
    on_floor = (np.abs(p[..., 0]) < 5.99) & (np.abs(p[..., 2]) < 5.99) & (t > 0)  # rays past the floor's edge miss it
    return KD / np.pi * I * S * np.abs(wi[..., 1:2]) / d2, keep & on_floor[..., None]


def check(got, want, keep, tol=2e-4):
    scale = float(np.max(want))
    assert scale > 0
    err = np.abs(got - want)[keep] / scale
    print("worst error %.2e relative to the brightest sample, %d of %d samples checked" % (float(err.max()), int(keep.sum()), keep.size))
    assert float(err.max()) <= tol


def gonio_S(img, w2l):
    def S(w):
        wl = w @ w2l[:3, :3].T
        wl = wl / np.linalg.norm(wl, axis=-1, keepdims=True)
        wp = np.stack([wl[..., 0], wl[..., 2], wl[..., 1]], -1)  # y and z swapped
        theta = np.arccos(np.clip(wp[..., 2], -1, 1))
        phi = np.mod(np.arctan2(wp[..., 1], wp[..., 0]), 2 * np.pi)
        keep = np.sin(theta) > 0.05  # phi is ill-conditioned at the poles
        return bilinear(img, phi / (2 * np.pi), theta / np.pi), np.broadcast_to(keep[..., None], keep.shape + (3,))
    return S


def proj_S(img, w2l, fov):
    hh, ww = img.shape[:2]
    a = ww / hh
    x1, y1 = (a, 1.0) if a > 1 else (1.0, 1.0 / a)
    ita = 1.0 / np.tan(np.radians(fov) / 2)

    def S(w):
        wl = w @ w2l[:3, :3].T
        z = wl[..., 2]
        front = z >= 1e-3
        zs = np.where(front, z, 1.0)
        x, y = ita * wl[..., 0] / zs, ita * wl[..., 1] / zs
        inside = front & (np.abs(x) <= x1) & (np.abs(y) <= y1)
        val = bilinear(img, (x + x1) / (2 * x1), (y + y1) / (2 * y1)) * inside[..., None]
        margin = 1e-3
        keep = ~front | ((np.abs(np.abs(x) - x1) > margin) & (np.abs(np.abs(y) - y1) > margin))
        return val, np.broadcast_to(keep[..., None], keep.shape + (3,))
    return S, x1, y1


def pow2_map(w, h, seed):
    rng = np.random.default_rng(seed)
    return (0.2 + rng.random((h, w, 3))).astype(np.float32)


INTEGRATORS = ["path", "direct", ("direct", "one"), "whitted"]
INTEGRATOR_IDS = ["path", "direct-all", "direct-one", "whitted"]


@pytest.mark.parametrize("sampler", ["sobol", "halton"])
@pytest.mark.parametrize("integrator", INTEGRATORS, ids=INTEGRATOR_IDS)
def test_goniometric_closed_form(oracle, integrator, sampler):
    img = pow2_map(32, 16, 3)
    l2w = turned(POS, 35.0, 20.0)
    h = floor_scene(lambda h: h.light_goniometric(I, texels=img, light_to_world=l2w), integrator=integrator, sampler=sampler)
    got, _ = render(h)
    o, d = camera_rays(h, oracle)
    want, keep = expectation(o, d, gonio_S(img, f32_inverse(l2w)))
    check(got, want, keep)


@pytest.mark.parametrize("integrator,sampler", [("path", "sobol"), ("whitted", "halton"), (("direct", "one"), "sobol")], ids=["path-sobol", "whitted-halton", "direct-one-sobol"])
@pytest.mark.parametrize("shape", [(32, 16), (16, 32)], ids=["aspect2", "aspect0.5"])
def test_projection_closed_form(oracle, shape, integrator, sampler):
    img = pow2_map(shape[0], shape[1], 4)
    l2w = scenes.projector_transform(POS, [0.8, 0.0, 1.6])
    h = floor_scene(lambda h: h.light_projection(I, img, fov=40.0, light_to_world=l2w), integrator=integrator, sampler=sampler)
    got, _ = render(h)
    o, d = camera_rays(h, oracle)
    S, _, _ = proj_S(img, f32_inverse(l2w), 40.0)
    want, keep = expectation(o, d, S)
    check(got, want, keep)
    dark = (want == 0) & keep
    assert dark.sum() > 0.02 * dark.size and np.all(got[dark] == 0)  # outside the frustum (the floor behind the projector included)
    assert (want > 0).sum() > 0.02 * want.size


def test_projection_behind_the_projector_is_black():
    img = pow2_map(16, 16, 6)
    l2w = scenes.projector_transform(POS, [0.0, 6.0, 0.5])  # aims straight up: the whole floor lies behind the hither plane
    got, st = render(floor_scene(lambda h: h.light_projection(I, img, fov=90.0, light_to_world=l2w)))
    assert np.all(got == 0) and st["shadow_rays"] == 0


@pytest.mark.parametrize("integrator", ["path", "direct"])
@pytest.mark.parametrize("sampler", ["sobol", "halton"])
def test_goniometric_without_map_is_a_point_light(integrator, sampler):
    l2w = turned(POS, 35.0, 20.0)
    a, sa = render(floor_scene(lambda h: h.light_goniometric(I, light_to_world=l2w), integrator=integrator, sampler=sampler))
    b, sb = render(floor_scene(lambda h: h.light_point(list(l2w[:3, 3].astype(np.float32)), I), integrator=integrator, sampler=sampler))
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
    assert all(sa[k] == sb[k] for k in ("rays", "closest_rays", "shadow_rays"))


def both_with_area(h, kind, img):
    """the image light beside a small emitting quad, so that the light distributions have two entries"""
    h.trianglemesh([0, 1, 2, 0, 2, 3], np.array([[-3, 3, 2], [-2, 3, 2], [-2, 3, 3], [-3, 3, 3]], np.float32), material=0, emit=[4.0, 4.0, 4.0])
    if kind == "goniometric":
        h.light_goniometric(I, texels=img, light_to_world=turned(POS, 35.0, 20.0))
    else:
        h.light_projection(I, img, fov=40.0, light_to_world=scenes.projector_transform(POS, [0.8, 0.0, 1.6]))


@pytest.mark.parametrize("strategy", ["uniform", "power", "spatial"])
@pytest.mark.parametrize("kind", ["goniometric", "projection"])
def test_mixed_with_an_area_light_renders(kind, strategy):
    """every strategy runs the light-level-2 kernels to the end with finite samples and lit pixels from both lights"""
    img = scenes.gonio_map() if kind == "goniometric" else scenes.projector_slide()  # non-power-of-two: the Lanczos zoom
    h = HostScene()
    h.material(_abi.MAT_MATTE, list(KD) + [0.0])
    h.trianglemesh(FLOOR_IDX, FLOOR, material=0)
    both_with_area(h, kind, img)
    h.look_at([0, 5, -5], [0, 0, 0.5], [0, 1, 0])
    h.film(24, 24)
    h.camera(fov=60.0)
    h.sampler(4)
    h.integrator(maxdepth=3, lightsamplestrategy=strategy)
    h.world_end()
    s, st = render(h)
    assert np.all(np.isfinite(s)) and float(s.mean()) > 0 and st["shadow_rays"] > 0


@pytest.mark.parametrize("lights", ["goniometric", "projection"])
@pytest.mark.parametrize("integrator", ["path", ("direct", "all"), ("direct", "one"), "whitted"], ids=["path", "direct-all", "direct-one", "whitted"])
def test_cornell_box_with_image_light(lights, integrator):
    h = scenes.cornell_box(xres=16, yres=16, spp=4, lights=lights, integrator=integrator, materials="mixed")
    s, st = render(h)
    assert np.all(np.isfinite(s)) and float(s.mean()) > 0 and st["shadow_rays"] > 0


@pytest.mark.parametrize("sampler", ["sobol", "halton"])
@pytest.mark.parametrize("kind", ["goniometric", "projection"])
def test_instanced_floor_closed_form(oracle, kind, sampler):
    """the instanced k_shade<2, *, true, 0> instantiations"""
    img = pow2_map(32, 16, 7)
    if kind == "goniometric":
        l2w = turned(POS, 35.0, 20.0)
        h = floor_scene(lambda h: h.light_goniometric(I, texels=img, light_to_world=l2w), sampler=sampler, instanced=True)
        S = gonio_S(img, f32_inverse(l2w))
    else:
        l2w = scenes.projector_transform(POS, [0.8, 0.0, 1.6])
        h = floor_scene(lambda h: h.light_projection(I, img, fov=40.0, light_to_world=l2w), sampler=sampler, instanced=True)
        S = proj_S(img, f32_inverse(l2w), 40.0)[0]
    got, _ = render(h)
    o, d = camera_rays(h, oracle)
    want, keep = expectation(o, d, S)
    check(got, want, keep)


# ---- power(): the power light distribution beside a point light ------------------------------------------------------------
# With lightsamplestrategy "power" every sample at maxdepth 1 is c_i / pmf_i for the light i its sample dimension chose, where
# pmf_i = y(power_i) / sum_j y(power_j) (lightdistrib.rs, integrator.rs:574-584).  power() is 4 pi I lookup((.5, .5), .5) for the
# goniometric light and 2 pi (1 - cos_total_width) I lookup((.5, .5), .5) for the projection light (goniometric.rs:266-280,
# projection.rs:379-398): width 0.5 is the bilinear lookup of pyramid level L - 2 (mipmap.rs:233-252, delta = 0).

P2 = np.array([-1.5, 3.0, 2.5])
I2 = np.array([12.0, 14.0, 9.0])


def y_of(rgb):
    return 0.212671 * rgb[0] + 0.715160 * rgb[1] + 0.072169 * rgb[2]


def lookup_half(img):
    """MipMap::lookup_pnt_flt((0.5, 0.5), 0.5) on a power-of-two map: the box pyramid with Repeat wrap, level L - 2"""
    levels = [img.astype(np.float64)]
    n_levels = 1 + int(np.floor(np.log2(max(img.shape[0], img.shape[1]))))
    for _ in range(1, n_levels):
        f = levels[-1]
        hh, ww = f.shape[:2]
        ch, cw = max(1, hh // 2), max(1, ww // 2)
        t, s_ = np.arange(ch)[:, None], np.arange(cw)[None, :]
        tx = lambda a, b: f[b % hh, a % ww]
        levels.append(0.25 * (tx(2 * s_, 2 * t) + tx(2 * s_ + 1, 2 * t) + tx(2 * s_, 2 * t + 1) + tx(2 * s_ + 1, 2 * t + 1)))
    return bilinear(levels[n_levels - 2], np.array(0.5), np.array(0.5))


@pytest.mark.parametrize("kind", ["goniometric", "projection"])
def test_power_strategy_pins_power(oracle, kind):
    img = pow2_map(32, 16, 11)
    img[:8, :16] *= 3.0  # a bright quadrant: the width-0.5 lookup averages it in, level 0 at the centre does not
    if kind == "goniometric":
        l2w = turned(POS, 35.0, 20.0)
        add = lambda h: h.light_goniometric(I, texels=img, light_to_world=l2w)
        S = gonio_S(img, f32_inverse(l2w))
        power = 4 * np.pi * I * lookup_half(img)
    else:
        fov = 40.0
        l2w = scenes.projector_transform(POS, [0.8, 0.0, 1.6])
        add = lambda h: h.light_projection(I, img, fov=fov, light_to_world=l2w)
        S, x1, y1 = proj_S(img, f32_inverse(l2w), fov)
        tan_half = np.tan(np.radians(fov) / 2)
        cos_total_width = 1.0 / np.sqrt(1.0 + (x1 * x1 + y1 * y1) * tan_half * tan_half)  # the corner of the screen window
        power = 2 * np.pi * (1 - cos_total_width) * I * lookup_half(img)

    def lights(h):
        add(h)
        h.light_point(P2, I2)

    h = floor_scene(lights, spp=8, strategy="power")
    got, _ = render(h)
    o, d = camera_rays(h, oracle)
    c_img, keep = expectation(o, d, S)
    t = -o[..., 1] / d[..., 1]
    p = o + d * t[..., None]
    v = P2 - p
    d2 = np.sum(v * v, -1, keepdims=True)
    c_pt = KD / np.pi * I2 * np.abs(v[..., 1:2] / np.sqrt(d2)) / d2
    w = np.array([y_of(power), y_of(4 * np.pi * I2)])
    pmf = w / w.sum()
    a, b = c_img / pmf[0], c_pt / pmf[1]
    scale = float(max(a.max(), b.max()))
    ea, eb = np.abs(got - a) / scale, np.abs(got - b) / scale
    ok_a, ok_b = np.all(ea <= 2e-4, -1), np.all(eb <= 2e-4, -1)
    k = keep[..., 0] & (np.abs(a - b).max(-1) > 1e-3 * scale)  # samples whose two candidates can be told apart
    print("%s: pmf %s; %d samples chose the image light, %d the point light, %d match neither"
          % (kind, pmf, int((ok_a & k).sum()), int((ok_b & k).sum()), int((k & ~ok_a & ~ok_b).sum())))
    assert np.all(ok_a[k] | ok_b[k])
    assert (ok_a & k).sum() > 0.1 * k.sum() and (ok_b & k).sum() > 0.1 * k.sum()
