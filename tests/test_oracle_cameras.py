"""The orthographic and environment cameras of tests/camera_ref (the oracle the GPU camera tests compare against) held to float64
closed forms derived here from the scene description alone: ray geometry, a lit quad's footprint, an environment map read through
the camera, the texture filter width each camera's differentials select, and the orthographic thin-lens differential as rs_pbrt
writes it.  CPU only."""
import numpy as np
import pytest

import camera_ref
import oracle_lib
from rs_pbrt_b200 import _abi
from rs_pbrt_b200.host import HostScene

f32 = np.float32


def model(h):
    return h.camera_model.contents


def look_basis(eye, look, up):
    """Transform::look_at in float64: camera x (left), y (up) and z (view) axes in world space."""
    eye, look, up = (np.asarray(v, np.float64) for v in (eye, look, up))
    d = (look - eye) / np.linalg.norm(look - eye)
    left = np.cross(up / np.linalg.norm(up), d)
    left /= np.linalg.norm(left)
    return left, np.cross(d, left), d


def ortho_point(pf, res, sw, eye, basis):
    """raster -> camera of an orthographic camera (the screen window spread over the full film) -> world, in float64."""
    xc = sw[0] + pf[..., 0] / res[0] * (sw[1] - sw[0])
    yc = sw[3] - pf[..., 1] / res[1] * (sw[3] - sw[2])
    return np.asarray(eye, np.float64) + xc[..., None] * basis[0] + yc[..., None] * basis[1]


def env_dir(pf, res):
    """EnvironmentCamera's camera-space direction in float64 (environment.rs:93-100)."""
    th = np.pi * pf[..., 1] / res[1]
    ph = 2.0 * np.pi * pf[..., 0] / res[0]
    return np.stack([np.sin(th) * np.cos(ph), np.cos(th), np.sin(th) * np.sin(ph)], -1)


def camera_samples(h, spp):
    """Every sample's CameraSample (p_film, time, p_lens) as the sampler draws it: (h, w, spp, 5)."""
    o = oracle_lib.OracleScene(h.desc)
    sb = h.params.contents.sample_bounds
    out = np.zeros((sb[3] - sb[1], sb[2] - sb[0], spp, 5), np.float64)
    for py in range(sb[1], sb[3]):
        for px in range(sb[0], sb[2]):
            for k in range(spp):
                out[py - sb[1], px - sb[0], k] = o.camera_sample(h.params, px, py, k)[:5]
    return out


# ---- orthographic camera over a lit Lambertian quad ---------------------------------------------------------------------------------

RES, SW, EYE = (32, 24), [-2.0, 2.0, -1.5, 1.5], [0.3, -0.2, -5.0]  # 8 raster pixels per unit both ways
QUAD = (-0.95, 1.05, -0.8, 1.1)  # x0, x1, y0, y1 at z = 0: every edge falls inside a pixel


def quad_scene(spp=16):
    h = HostScene()
    m = h.material(_abi.MAT_MATTE, [0.5, 0.5, 0.5, 0.0])
    x0, x1, y0, y1 = QUAD
    P = np.array([[x0, y0, 0], [x1, y0, 0], [x1, y1, 0], [x0, y1, 0]], f32)
    h.trianglemesh(np.array([0, 1, 2, 0, 2, 3], np.uint32), P, material=m)
    h.light_distant([0.0, 0.0, -1.0], [0.0, 0.0, 0.0], [1.0, 1.0, 1.0])  # arrives along +z: cos = 1 on the quad
    h.look_at(EYE, [EYE[0], EYE[1], 0.0], [0, 1, 0])
    h.film(*RES)
    h.camera_orthographic(screenwindow=SW)
    h.sampler(spp)
    h.integrator(maxdepth=1, lightsamplestrategy="uniform")
    h.world_end(n_threads=1)
    return h


def test_orthographic_rays_are_parallel_to_the_view_axis():
    eye, look, up = [1.0, 2.0, -4.0], [0.2, 0.5, 3.0], [0.1, 1.0, 0.2]
    h = HostScene()
    h.trianglemesh(np.array([0, 1, 2], np.uint32), np.array([[0, 0, 5], [1, 0, 5], [0, 1, 5]], f32), material=h.material(_abi.MAT_MATTE, [0.5] * 3 + [0.0]))
    h.light_point([0, 0, 0], [1, 1, 1])
    h.look_at(eye, look, up)
    h.film(24, 16)
    h.camera_orthographic(screenwindow=[-3.0, 3.0, -2.0, 2.0])
    h.sampler(1)
    h.integrator(maxdepth=1)
    h.world_end(n_threads=1)
    rng = np.random.default_rng(1)
    pf = rng.uniform(0.0, [24.0, 16.0], (500, 2))
    r = camera_ref.camera_rays(h.desc.contents.camera, model(h), pf, 0.5, [0.5, 0.5])
    basis = look_basis(eye, look, up)
    np.testing.assert_allclose(r["d"], np.broadcast_to(basis[2], (500, 3)), atol=2e-6)
    np.testing.assert_allclose(r["o"], ortho_point(pf, (24, 16), [-3.0, 3.0, -2.0, 2.0], eye, basis), atol=2e-5)
    # no lens: the differentials are the origin one raster step over, along the same direction (orthographic.rs:212-220)
    assert r["has_diff"].all()
    np.testing.assert_allclose(r["rx_o"] - r["o"], np.broadcast_to(basis[0] * 6.0 / 24, (500, 3)), atol=2e-5)
    np.testing.assert_allclose(r["ry_o"] - r["o"], np.broadcast_to(-basis[1] * 4.0 / 16, (500, 3)), atol=2e-5)
    assert np.array_equal(r["rx_d"], r["d"]) and np.array_equal(r["ry_d"], r["d"])


def test_orthographic_samples_hit_where_the_raster_maps():
    """Each sample's radiance is Kd/pi * L where raster_to_camera(p_film) through camera_to_world lies on the quad, and 0 elsewhere."""
    spp = 16
    h = quad_scene(spp)
    cs = camera_samples(h, spp)
    _, got, _, _ = camera_ref.CameraScene(h.desc, model(h)).render(h.params)
    w = ortho_point(cs[..., 0:2], RES, SW, EYE, look_basis(EYE, [EYE[0], EYE[1], 0.0], [0, 1, 0]))
    x0, x1, y0, y1 = QUAD
    inside = (w[..., 0] > x0) & (w[..., 0] < x1) & (w[..., 1] > y0) & (w[..., 1] < y1)
    margin = np.minimum.reduce([np.abs(w[..., 0] - x0), np.abs(w[..., 0] - x1), np.abs(w[..., 1] - y0), np.abs(w[..., 1] - y1)])
    sure = margin > 1e-4
    exp = np.where(inside, 0.5 / np.pi, 0.0)[..., None]
    np.testing.assert_allclose(got[sure], np.broadcast_to(exp, got.shape)[sure], rtol=2e-6, atol=0)
    assert inside.sum() > 1000 and (~inside).sum() > 1000


def test_orthographic_footprint_is_area_times_raster_density():
    spp = 16
    h = quad_scene(spp)
    _, got, _, _ = camera_ref.CameraScene(h.desc, model(h)).render(h.params)
    covered = float((got[..., 0] > 0).sum()) / spp  # pixels
    x0, x1, y0, y1 = QUAD
    density = (RES[0] / (SW[1] - SW[0])) * (RES[1] / (SW[3] - SW[2]))
    assert abs(covered - (x1 - x0) * (y1 - y0) * density) < 1.5, covered


# ---- environment camera inside a direction-encoding environment map -----------------------------------------------------------------

def encoding_map(w=64, h=32):
    jj, ii = np.mgrid[0:h, 0:w]
    u, v = (ii + 0.5) / w, (jj + 0.5) / h
    return np.stack([0.5 + 0.4 * np.cos(2 * np.pi * u), v, 0.3 + 0.6 * ((ii * 5 + jj * 3) % 7) / 7.0], -1).astype(f32)


def bilerp_repeat(img, s, t):
    """MipMap level-0 `triangle` lookup with ImageWrap::Repeat (mipmap.rs:323-336), in float64."""
    H, W = img.shape[:2]
    x, y = s * W - 0.5, t * H - 0.5
    x0, y0 = np.floor(x).astype(np.int64), np.floor(y).astype(np.int64)
    dx, dy = (x - x0)[..., None], (y - y0)[..., None]
    tex = lambda i, j: img[j % H, i % W].astype(np.float64)  # noqa: E731
    return (1 - dx) * (1 - dy) * tex(x0, y0) + (1 - dx) * dy * tex(x0, y0 + 1) + dx * (1 - dy) * tex(x0 + 1, y0) + dx * dy * tex(x0 + 1, y0 + 1)


@pytest.mark.parametrize("crop", [None, [0.25, 0.75, 0.0, 0.5]], ids=["full", "crop"])
def test_environment_camera_reads_the_map_at_the_closed_form_direction(crop):
    """With a crop window too: the directions still divide by the full film resolution."""
    res, spp = (64, 32), 8
    img = encoding_map()
    h = HostScene()
    far = np.array([0.0, -30.0, -100.0])  # one small triangle (a scene needs geometry), well away from the seams and poles checked
    h.trianglemesh(np.array([0, 1, 2], np.uint32), (far + np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0]])).astype(f32), material=h.material(_abi.MAT_MATTE, [0.5] * 3 + [0.0]))
    h.light_infinite([1.0, 1.0, 1.0], texels=img)
    h.look_at([0, 0, 0], [0, 0, 1], [0, 1, 0])  # camera_to_world = identity
    h.film(*res, crop=crop)
    h.camera_environment()
    h.sampler(spp)
    h.integrator(maxdepth=1, lightsamplestrategy="uniform")
    h.world_end(n_threads=1)
    assert np.array_equal(np.array(h.desc.contents.camera.camera_to_world).reshape(4, 4), np.eye(4))
    cs = camera_samples(h, spp)
    _, got, _, _ = camera_ref.CameraScene(h.desc, model(h)).render(h.params)
    pf = cs[..., 0:2]
    d = env_dir(pf, res)
    # InfiniteAreaLight::le (infinite.rs): spherical_phi / spherical_theta of the light-space direction (identity here), z up
    s = np.mod(np.arctan2(d[..., 1], d[..., 0]), 2 * np.pi) / (2 * np.pi)
    t = np.arccos(np.clip(d[..., 2], -1, 1)) / np.pi
    exp = bilerp_repeat(img, s, t)
    away = np.degrees(np.arccos(np.clip(d @ (far / np.linalg.norm(far)), -1, 1))) > 5.0
    ok = away & (np.abs(d[..., 2]) < 0.999)  # (the light's own poles: its phi is atan2 of two rounding residues there)
    np.testing.assert_allclose(got[ok], exp[ok], rtol=0, atol=1e-4)
    if crop is not None:
        assert ok.sum() > 1000
        return
    # the camera's seam (p_film.x at 0 and at the full width), its poles (p_film.y at 0 and at the full height) and the light's seam
    for region in (pf[..., 0] < 0.5, pf[..., 0] > res[0] - 0.5, pf[..., 1] < 0.5, pf[..., 1] > res[1] - 0.5, (s < 0.01) | (s > 0.99)):
        assert (region & ok).sum() >= 8
    # phi and theta swapped would read elsewhere
    ds = env_dir(pf[..., ::-1] * np.array([res[0] / res[1], res[1] / res[0]]), res)
    swapped = bilerp_repeat(img, np.mod(np.arctan2(ds[..., 1], ds[..., 0]), 2 * np.pi) / (2 * np.pi), np.arccos(np.clip(ds[..., 2], -1, 1)) / np.pi)
    assert np.abs(swapped[ok] - got[ok]).max() > 0.1


# ---- texture filter width of each camera -------------------------------------------------------------------------------------------

S_PLANE, SCALE = 40.0, 6.0


def plane_scene(kind, texels=None, spp=4, res=32, half=20.0):
    """A large vertical matte plane (z = 0, uv over [-S, S]^2) under a constant white InfiniteAreaLight, maxdepth 1: every sample's
    radiance is Kd(hit) times a lighting estimate that does not depend on Kd, so textured / constant isolates the filtered texel."""
    h = HostScene()
    if texels is None:
        m = h.material(_abi.MAT_MATTE, [0.5, 0.5, 0.5, 0.0])
    else:
        tex = h.texture_image(texels[::-1], trilinear=True, uscale=SCALE, vscale=SCALE)  # (the call flips y; texels[j] is row t = j)
        m = h.material(_abi.MAT_MATTE, [0.5, 0.5, 0.5, 0.0], textures={0: tex})
    h.light_infinite([1.0, 1.0, 1.0])
    S = S_PLANE
    P = np.array([[-S, -S, 0], [S, -S, 0], [S, S, 0], [-S, S, 0]], f32)
    UV = np.array([[0, 0], [1, 0], [1, 1], [0, 1]], f32)
    h.trianglemesh(np.array([0, 1, 2, 0, 2, 3], np.uint32), P, UV=UV, material=m)
    h.look_at([0.5, 0.3, -9.0], [0.5, 0.3, 0.0], [0, 1, 0])
    h.film(res, res)
    if kind == "orthographic":
        h.camera_orthographic(screenwindow=[-half, half, -half, half])
    else:
        h.camera_environment()
    h.sampler(spp)
    h.integrator(maxdepth=1, lightsamplestrategy="uniform")
    h.world_end(n_threads=1)
    return h


def blocky_image():
    rng = np.random.default_rng(7)
    return (np.kron(rng.random((16, 16, 3)), np.ones((4, 4, 1))) * 0.8 + 0.1).astype(f32)  # 64x64: levels differ visibly


@pytest.mark.parametrize("kind", ["orthographic", "environment"])
def test_first_hit_filter_width(kind):
    """Orthographic: the trilinear width is SCALE * |dx_camera| / sqrt(spp) / (2 S) at every sample (the differentials are the origin
    one raster step over, along the view axis, on a plane facing the camera).  Environment: no differential, so every first-hit
    lookup is the level-0 bilinear one."""
    spp, res, half = 4, 32, 20.0
    img = blocky_image()
    ht, hc = plane_scene(kind, img, spp, res, half), plane_scene(kind, None, spp, res, half)
    _, tex_s, _, _ = camera_ref.CameraScene(ht.desc, model(ht)).render(ht.params)
    _, lit_s, _, _ = camera_ref.CameraScene(hc.desc, model(hc)).render(hc.params)
    cs = camera_samples(ht, spp)
    eye = np.array([0.5, 0.3, -9.0])
    if kind == "orthographic":
        P = ortho_point(cs[..., 0:2], (res, res), [-half, half, -half, half], eye, look_basis(eye, [0.5, 0.3, 0.0], [0, 1, 0]))
    else:
        d = env_dir(cs[..., 0:2], (res, res))  # camera_to_world's rotation is the identity here
        P = eye + d * np.where(d[..., 2:3] > 1e-3, -eye[2] / np.maximum(d[..., 2:3], 1e-3), np.nan)
    uv = (P[..., 0:2] + S_PLANE) / (2 * S_PLANE)
    texture = oracle_lib.OracleTexture(img, trilinear=True)
    ok = (lit_s[..., 0] > 0) & np.isfinite(uv).all(-1) & (np.abs(P[..., 0:2]) < S_PLANE - 1).all(-1)
    if kind == "environment":
        ok &= np.abs(P[..., 0:2] - eye[0:2]).max(-1) < 12.0  # (far off the axis the f32 hit point drifts by more than a texel's fraction)
    got = tex_s[ok] / lit_s[ok] * 0.5
    st = uv[ok] * SCALE
    if kind == "orthographic":
        width = SCALE * ((2 * half / res) / np.sqrt(spp)) / (2 * S_PLANE)
        exp = texture.lookup(st, dst0=np.tile([[width, 0.0]], (len(st), 1)))
        level0 = texture.lookup(st)
        assert np.abs(level0 - got).max() > 0.05  # the filtered value is not the level-0 one
    else:
        exp = texture.lookup(st)
    np.testing.assert_allclose(got, exp, rtol=0, atol=4e-3)
    assert ok.sum() > 300


# ---- orthographic thin lens: the differential as rs_pbrt writes it ----------------------------------------------------------------

def concentric(u):
    ux, uy = 2 * u[0] - 1, 2 * u[1] - 1
    if ux == 0 and uy == 0:
        return np.zeros(2)
    if abs(ux) > abs(uy):
        r, th = ux, (np.pi / 4) * (uy / ux)
    else:
        r, th = uy, np.pi / 2 - (np.pi / 4) * (ux / uy)
    return r * np.array([np.cos(th), np.sin(th)])


def test_orthographic_thin_lens_differential_quirk():
    """orthographic.rs:177-211 in float64: the ray leaves the lens point towards p_camera + (0, 0, focal_distance); both differentials
    leave the same lens point towards ONE focus point, p_camera + dx_camera + (0, 0, focal_distance / d.z) with the refracted d, so
    ry == rx and dy_camera never enters (pbrt-v3 would aim ry at p_camera + dy_camera)."""
    lr, fd, res, sw, spp = 0.4, 7.0, (20, 16), [-2.5, 2.5, -2.0, 2.0], 4
    eye, look, up = [0.2, 1.0, -6.0], [0.0, 0.4, 2.0], [0.0, 1.0, 0.1]
    h = HostScene()
    h.trianglemesh(np.array([0, 1, 2], np.uint32), np.array([[0, 0, 5], [1, 0, 5], [0, 1, 5]], f32), material=h.material(_abi.MAT_MATTE, [0.5] * 3 + [0.0]))
    h.light_point([0, 0, 0], [1, 1, 1])
    h.look_at(eye, look, up)
    h.film(*res)
    h.camera_orthographic(lensradius=lr, focaldistance=fd, screenwindow=sw)
    h.sampler(spp)
    h.integrator(maxdepth=1)
    h.world_end(n_threads=1)
    rng = np.random.default_rng(5)
    n = 300
    pf = rng.uniform(0.0, res, (n, 2))
    ul = rng.uniform(0.02, 0.98, (n, 2))
    r = camera_ref.camera_rays(h.desc.contents.camera, model(h), pf, 0.5, ul, spp=spp)
    basis = np.stack(look_basis(eye, look, up), 1)  # camera -> world rotation
    dxc = np.array([(sw[1] - sw[0]) / res[0], 0.0, 0.0])
    dyc = np.array([0.0, -(sw[3] - sw[2]) / res[1], 0.0])
    s = 1.0 / np.sqrt(spp)
    assert r["has_diff"].all()
    assert np.array_equal(r["rx_d"], r["ry_d"]) and np.array_equal(r["rx_o"], r["ry_o"])
    for i in range(n):
        pc = np.array([sw[0] + pf[i, 0] / res[0] * (sw[1] - sw[0]), sw[3] - pf[i, 1] / res[1] * (sw[3] - sw[2]), 0.0])
        pl = np.append(concentric(ul[i]) * lr, 0.0)
        d = pc + np.array([0.0, 0.0, fd]) - pl
        d /= np.linalg.norm(d)
        rd = pc + dxc + np.array([0.0, 0.0, fd / d[2]]) - pl
        rd /= np.linalg.norm(rd)
        dw, rdw = basis @ d, basis @ rd
        np.testing.assert_allclose(r["d"][i], dw, atol=3e-6)
        np.testing.assert_allclose(r["rx_d"][i], dw + (rdw - dw) * s, atol=3e-6)
        # pbrt-v3's ry (focus point from dy_camera) would differ
        ry3 = pc + dyc + np.array([0.0, 0.0, fd / d[2]]) - pl
        ry3 = basis @ (ry3 / np.linalg.norm(ry3))
        assert np.abs(r["ry_d"][i] - (dw + (ry3 - dw) * s)).max() > 1e-3
