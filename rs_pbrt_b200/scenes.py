"""Seeded synthetic stand-ins for BASELINE.json's configs (SURVEY.md section 8d).

The reference's test scenes live in an external repository that is not available offline, so every
config is generated procedurally, in world space, and fed through the same HostScene calls a .pbrt
file would produce (Material / Shape "trianglemesh" / AreaLightSource / LookAt / Camera / Film /
Sampler "sobol" / Integrator "path").  Only numpy is used here; all rendering numerics are in the
C++/CUDA library.
"""
import numpy as np

from . import _abi
from .host import HostScene


def _quad(p0, p1, p2, p3):
    """Two triangles (0,1,2) (0,2,3) over four corners."""
    P = np.array([p0, p1, p2, p3], np.float32)
    idx = np.array([0, 1, 2, 0, 2, 3], np.uint32)
    return idx, P


def _box(corners_bottom, height_pts):
    """Closed prism from a bottom quadrilateral (4x3) and its top quadrilateral (4x3): 5 visible faces, 10 triangles."""
    b = np.asarray(corners_bottom, np.float32)
    t = np.asarray(height_pts, np.float32)
    P = np.concatenate([b, t], 0)
    faces = [(4, 5, 6, 7)]  # top
    for i in range(4):
        j = (i + 1) % 4
        faces.append((i, j, 4 + j, 4 + i))
    idx = []
    for a, b_, c, d in faces:
        idx += [a, b_, c, a, c, d]
    return np.array(idx, np.uint32), P


def cornell_box(xres=400, yres=400, spp=64, maxdepth=5, strategy="spatial", filter="box", xwidth=0.5, ywidth=0.5, lensradius=0.0,
                focaldistance=1e6, n_threads=8, crop=None, materials="matte", lights="area", sampler="sobol", samplepixelcenter=False, integrator="path", textures=None, lightsamples=1,
                alpha=None, quantize_textures=False, camera_end=None, shutter=(0.0, 1.0), transform_times=(0.0, 1.0)):
    """Canonical Cornell box: 5 walls, short and tall block, ceiling light quad (2 triangles => 2 area lights, so
    the spatial light distribution is active).  32 triangles.  `materials="mixed"` swaps the blocks to glass /
    metal and the floor to plastic for BxDF coverage ("translucent", "mix": TranslucentMaterial / MixMaterial on blocks, floor and back wall).  `lights`: "area" (the ceiling quad only), "delta" (plus a point, a spot
    and a distant LightSource, declared before / between / after the shapes so the scene.lights order is interleaved),
    "point" / "spot" / "distant" (that single delta light and no emitter).  `textures`: None, "ewa" or "trilinear" -- image textures
    (imagemap.rs) on the floor (matte Kd: a checker of a non-power-of-two resolution, repeated), the back wall (matte Kd: noise,
    clamped, with a uv offset), the short block (plastic Kd and Ks) and the tall block (uber Kd and opacity, some texels opaque
    black / fully transparent so that the lobe list changes from hit to hit).  `alpha`: None, or "masks" -- three cards hang in the box with
    the Shape's "alpha" / "shadowalpha" float textures (triangle.rs:313-330,593-654): a leaf-like cut-out through an image mask (visible
    and shadow-casting only where the mask is non-zero), a card with a shadow-alpha mask only (fully visible, casts a shadow with holes)
    and a card with `"float alpha" 0` (never hit by anything).  `quantize_textures`: every image texel is rounded to a multiple of 1/255, so
    that the scene equals its own .pbrt export (rs_pbrt reads images as 8-bit RGB; rs_pbrt_b200/pbrt_export.py)."""
    h = HostScene()
    if quantize_textures:
        _ti = h.texture_image
        h.texture_image = lambda rgb, **kw: _ti((np.round(np.clip(np.asarray(rgb, np.float32), 0.0, 1.0) * 255.0) / 255.0).astype(np.float32), **kw)
    if lightsamples != 1:
        h.light_samples(lightsamples)  # "nsamples" of every light below (DirectLightingIntegrator "all")
    if lights in ("delta", "point"):
        h.light_point([278.0, 420.0, 279.5], [30000.0, 30000.0, 24000.0], scale=[1.5, 1.5, 1.5])
    white = h.material(_abi.MAT_MATTE, [0.73, 0.73, 0.73, 0.0])
    red = h.material(_abi.MAT_MATTE, [0.65, 0.05, 0.05, 0.0])
    green = h.material(_abi.MAT_MATTE, [0.12, 0.45, 0.15, 0.0])
    light_m = h.material(_abi.MAT_MATTE, [0.78, 0.78, 0.78, 0.0])
    short_m = tall_m = floor_m = white
    if materials == "mixed":
        floor_m = h.material(_abi.MAT_PLASTIC, [0.5, 0.5, 0.5, 0.3, 0.3, 0.3, 0.1, 1.0])
        short_m = h.material(_abi.MAT_GLASS, [1, 1, 1, 1, 1, 1, 1.5, 0.0, 0.0, 1.0])
        tall_m = h.material(_abi.MAT_METAL, [0.2, 0.92, 1.1, 3.9, 2.45, 2.14, 0.05, 0.05, 1.0])
    elif materials == "translucent":  # TranslucentMaterial (translucent.rs): all four lobes on the short block, diffuse-only / transmit-only variants elsewhere
        short_m = h.material(_abi.MAT_TRANSLUCENT, [0.6, 0.5, 0.3, 0.3, 0.3, 0.3, 0.5, 0.5, 0.5, 0.5, 0.5, 0.5, 0.15, 1.0])
        tall_m = h.material(_abi.MAT_TRANSLUCENT, [0.25, 0.4, 0.6, 0.0, 0.0, 0.0, 0.3, 0.3, 0.3, 0.7, 0.7, 0.7, 0.1, 1.0])
        floor_m = h.material(_abi.MAT_TRANSLUCENT, [0.5, 0.5, 0.5, 0.25, 0.25, 0.25, 1.0, 1.0, 1.0, 0.0, 0.0, 0.0, 0.2, 0.0])
    back_m = white
    ceil_m, left_m, right_m = white, red, green
    if callable(materials):  # materials(h) -> {"floor" | "short" | "tall" | "back" | "ceiling" | "left" | "right": material index}: the randomised scenes of tests/test_emu_kernels.py
        chosen = materials(h)
        floor_m, short_m, tall_m, back_m = (chosen.get(k, white) for k in ("floor", "short", "tall", "back"))
        ceil_m, left_m, right_m = chosen.get("ceiling", white), chosen.get("left", red), chosen.get("right", green)
    if materials == "mix":  # MixMaterial (mixmat.rs): every lobe kind under an sc_opt scale, an amount outside [0, 1], a mix of a mix
        mirror = h.material(_abi.MAT_MIRROR, [0.9, 0.9, 0.9])
        short_m = h.material_mix(red, mirror, [1.2, 0.5, 0.0])  # Lambert + specular reflection; s1 = (1.2, .5, 0), s2 = clamp(1 - s1) = (0, .5, 1)
        plastic = h.material(_abi.MAT_PLASTIC, [0.3, 0.4, 0.5, 0.3, 0.3, 0.3, 0.1, 1.0])
        glass = h.material(_abi.MAT_GLASS, [1, 1, 1, 1, 1, 1, 1.5, 0.0, 0.0, 1.0])
        tall_m = h.material_mix(plastic, glass, [0.4, 0.4, 0.4])  # Lambert + microfacet + FresnelSpecular (direct / whitted: reflection + transmission lobes)
        metal = h.material(_abi.MAT_METAL, [0.2, 0.92, 1.1, 3.9, 2.45, 2.14, 0.05, 0.08, 1.0])
        inner = h.material_mix(green, metal, [0.6, 0.6, 0.6])
        substrate = h.material(_abi.MAT_SUBSTRATE, [0.4, 0.3, 0.2, 0.1, 0.1, 0.1, 0.1, 0.15, 1.0])
        floor_m = h.material_mix(inner, substrate, [0.25, 0.5, 0.75])  # the inner mix ignores the scale handed down (mixmat.rs:48), FresnelBlend takes s2
        translucent = h.material(_abi.MAT_TRANSLUCENT, [0.6, 0.5, 0.3, 0.3, 0.3, 0.3, 0.5, 0.5, 0.5, 0.5, 0.5, 0.5, 0.15, 1.0])
        oren = h.material(_abi.MAT_MATTE, [0.5, 0.6, 0.7, 25.0])
        back_m = h.material_mix(translucent, oren, [0.5, 0.5, 0.5])  # five lobes: Lambert R / T, microfacet R / T, Oren-Nayar
    if textures:
        tri = textures.startswith("trilinear")
        with_float = "+float" in textures  # also ImageTexture<Float> on sigma / roughness (roughness_to_alpha per hit)
        with_graph = "+graph" in textures  # also ConstantTexture / ScaleTexture / MixTexture nodes over the images
        with_bump = "+bump" in textures    # also "bumpmap" float textures (Material::bump) on the floor, the back wall and the tall block
        rng = np.random.default_rng(5)
        yy, xx = np.mgrid[0:20, 0:24]
        checker = np.where(((xx // 3 + yy // 2) % 2)[..., None] == 0, [0.8, 0.75, 0.7], [0.15, 0.2, 0.3]).astype(np.float32)
        t_floor = h.texture_image(checker, trilinear=tri, wrap=_abi.WRAP_REPEAT, uscale=3.0, vscale=2.0, gamma=True)
        noise = (0.2 + 0.6 * rng.random((32, 32, 3))).astype(np.float32)
        t_back = h.texture_image(noise, trilinear=tri, max_anisotropy=4.0, wrap=_abi.WRAP_CLAMP, uscale=1.5, vscale=1.5, udelta=-0.2, vdelta=0.1)
        stripes = np.zeros((8, 16, 3), np.float32)
        stripes[:, ::2] = [0.7, 0.3, 0.1]
        t_kd = h.texture_image(stripes, trilinear=tri, wrap=_abi.WRAP_BLACK, uscale=2.0, vscale=2.0)
        t_ks = h.texture_image((0.5 * rng.random((16, 16, 3))).astype(np.float32), trilinear=tri, scale=0.8)
        holes = np.ones((16, 16, 3), np.float32)
        holes[4:8, 4:12] = 0.0
        holes[10:13, 2:6] = 0.5
        t_op = h.texture_image(holes, trilinear=tri, wrap=_abi.WRAP_REPEAT, uscale=2.0, vscale=3.0)
        if with_graph:
            tint = h.texture_constant([0.9, 0.6, 0.4])
            amt = h.texture_image((rng.random((8, 8, 3))).astype(np.float32), trilinear=tri, float_valued=True, uscale=2.0)
            t_floor = h.texture_mix(h.texture_scale(t_floor, tint), t_floor, amt)           # mix(scale(checker, tint), checker, amount image)
            t_ks = h.texture_scale(t_ks, h.texture_scale(h.texture_constant([0.5, 0.5, 2.0]), t_ks))  # a three-level product
        floor_m = h.material(_abi.MAT_MATTE, [0.5, 0.5, 0.5, 0.0], textures={0: t_floor})
        back_m = h.material(_abi.MAT_MATTE, [0.5, 0.5, 0.5, 25.0], textures={0: t_back})
        short_m = h.material(_abi.MAT_PLASTIC, [0.5, 0.5, 0.5, 0.3, 0.3, 0.3, 0.1, 1.0], textures={0: t_kd, 1: t_ks})
        tall_p = np.zeros(19, np.float32)
        tall_p[0:3] = 0.4; tall_p[3:6] = 0.3; tall_p[6:9] = 0.1; tall_p[9:12] = 0.0; tall_p[12:15] = 1.0
        tall_p[15] = 0.05; tall_p[16] = 0.08; tall_p[17] = 1.5; tall_p[18] = 1.0
        tall_m = h.material(_abi.MAT_UBER, tall_p, textures={0: t_back, 4: t_op})
        if with_float:
            t_sig = h.texture_image((rng.random((8, 8, 3)) * np.where(rng.random((8, 8, 1)) < 0.3, 0.0, 1.0)).astype(np.float32), trilinear=tri, scale=60.0,
                                    float_valued=True)  # sigma in [0, 60) degrees, exactly 0 (=> Lambertian lobe) on some texels
            t_rough = h.texture_image((0.02 + 0.5 * rng.random((16, 8, 3))).astype(np.float32), trilinear=tri, uscale=2.0, float_valued=True)
            back_m = h.material(_abi.MAT_MATTE, [0.5, 0.5, 0.5, 25.0], textures={0: t_back, 1: t_sig})
            short_m = h.material(_abi.MAT_PLASTIC, [0.5, 0.5, 0.5, 0.3, 0.3, 0.3, 0.1, 1.0], textures={0: t_kd, 1: t_ks, 2: t_rough})
            tall_m = h.material(_abi.MAT_UBER, tall_p, textures={0: t_back, 4: t_op, 5: t_rough})
        if with_bump:
            rb = np.random.default_rng(21)
            bump_img = np.kron(rb.random((8, 8, 1)), np.ones((2, 2, 3))).astype(np.float32)
            t_bump = h.texture_image(bump_img, trilinear=tri, float_valued=True, uscale=3.0, vscale=3.0, scale=4.0)
            t_bump2 = h.texture_scale(t_bump, h.texture_constant([0.5], float_valued=True))
            floor_m = h.material(_abi.MAT_MATTE, [0.5, 0.5, 0.5, 0.0], textures={0: t_floor}, bump=t_bump)
            back_m = h.material(_abi.MAT_MATTE, [0.6, 0.6, 0.6, 0.0], bump=t_bump2)  # a bump map alone: constant Kd
            tall_m = h.material(_abi.MAT_PLASTIC, [0.3, 0.3, 0.5, 0.4, 0.4, 0.4, 0.08, 1.0], textures={1: t_ks}, bump=t_bump)
    W = 555.0
    h.trianglemesh(*_quad([W, 0, 0], [0, 0, 0], [0, 0, W], [W, 0, W]), material=floor_m)           # floor
    h.trianglemesh(*_quad([W, W, 0], [W, W, W], [0, W, W], [0, W, 0]), material=ceil_m)            # ceiling
    h.trianglemesh(*_quad([W, 0, W], [0, 0, W], [0, W, W], [W, W, W]), material=back_m)            # back wall
    h.trianglemesh(*_quad([0, 0, W], [0, 0, 0], [0, W, 0], [0, W, W]), material=right_m)           # right wall
    h.trianglemesh(*_quad([W, 0, 0], [W, 0, W], [W, W, W], [W, W, 0]), material=left_m)            # left wall
    if lights in ("delta", "spot"):
        h.light_spot([60.0, 520.0, 60.0], [300.0, 0.0, 300.0], [250000.0, 220000.0, 200000.0], coneangle=32.0, conedeltaangle=9.0)
    sb = [[130, 0, 65], [82, 0, 225], [240, 0, 272], [290, 0, 114]]
    st = [[x, 165.0, z] for x, _, z in sb]
    h.trianglemesh(*_box(sb, st), material=short_m)
    tb = [[423, 0, 247], [265, 0, 296], [314, 0, 456], [472, 0, 406]]
    tt = [[x, 330.0, z] for x, _, z in tb]
    h.trianglemesh(*_box(tb, tt), material=tall_m)
    if alpha:
        ra = np.random.default_rng(17)
        uvq = np.array([[0, 0], [1, 0], [1, 1], [0, 1]], np.float32)
        yy, xx = np.mgrid[0:24, 0:24]
        leaf = ((xx - 11.5) ** 2 / 130.0 + (yy - 11.5) ** 2 / 60.0 < 1.0).astype(np.float32)
        leaf[(xx + yy) % 7 == 0] = 0.0  # slits
        leaf = leaf * (0.3 + 0.7 * ra.random((24, 24))).astype(np.float32)  # non-zero values other than 1 count as opaque
        t_leaf = h.texture_image(np.repeat(leaf[..., None], 3, axis=2), float_valued=True, wrap=_abi.WRAP_CLAMP)
        holes2 = (ra.random((6, 10)) > 0.4).astype(np.float32)
        t_holes = h.texture_image(np.repeat(holes2[..., None], 3, axis=2), float_valued=True, uscale=2.0, vscale=2.0)
        t_zero = h.texture_constant([0.0], float_valued=True)
        card_m = h.material(_abi.MAT_MATTE, [0.2, 0.6, 0.25, 0.0])
        i1, P1 = _quad([120, 200, 150], [330, 230, 120], [330, 420, 180], [120, 390, 210])
        m1 = h.trianglemesh(i1, P1, UV=uvq, material=card_m)
        h.mesh_alpha(m1, alpha=t_leaf)
        i2, P2 = _quad([300, 300, 300], [500, 300, 330], [500, 430, 380], [300, 430, 350])
        m2 = h.trianglemesh(i2, P2, UV=uvq, material=card_m)
        h.mesh_alpha(m2, shadow_alpha=t_holes)
        i3, P3 = _quad([100, 100, 100], [450, 100, 100], [450, 450, 100], [100, 450, 100])
        m3 = h.trianglemesh(i3, P3, material=red)
        h.mesh_alpha(m3, alpha=t_zero, shadow_alpha=t_holes)
    ly = W - 1.0
    h.trianglemesh(*_quad([343, ly, 227], [343, ly, 332], [213, ly, 332], [213, ly, 227]), material=light_m,
                   emit=[17.0, 12.0, 4.0] if lights in ("area", "delta") else None)
    if lights in ("delta", "distant"):
        h.light_distant([0.3, 1.0, -1.5], [0.0, 0.0, 0.0], [1.5, 1.4, 1.1])  # shines in through the open front
    h.look_at([278, 273, -800], [278, 273, 0], [0, 1, 0])
    _camera_motion(h, camera_end, transform_times)
    h.film(xres, yres, crop=crop, filter=filter, xwidth=xwidth, ywidth=ywidth)
    h.camera(fov=39.3077, lensradius=lensradius, focaldistance=focaldistance, shutteropen=shutter[0], shutterclose=shutter[1])
    h.sampler(spp, name=sampler, samplepixelcenter=samplepixelcenter)
    _set_integrator(h, integrator, maxdepth, strategy)
    h.world_end(n_threads=n_threads)
    return h


def look_at_matrix(eye, look, up):
    """camera_to_world of `LookAt eye look up` (Transform::look_at, transform.rs:414-451), f32, row-major 4x4."""
    eye, look, up = (np.asarray(v, np.float32) for v in (eye, look, up))
    d = look - eye
    d = d / np.sqrt(np.sum(d * d))
    u = up / np.sqrt(np.sum(up * up))
    left = np.cross(u, d)
    left = left / np.sqrt(np.sum(left * left))
    m = np.eye(4, dtype=np.float32)
    m[:3, 0], m[:3, 1], m[:3, 2], m[:3, 3] = left, np.cross(d, left), d, eye
    return m


def _camera_motion(h, camera_end, transform_times):
    """An animated camera: `camera_end` is camera_to_world at the end time (None: static camera, nothing is declared)."""
    if camera_end is None:
        return
    h.transform_times(*transform_times)
    h.camera_motion(camera_end)


def motion_cornell(xres=64, yres=64, spp=16, dolly=150.0, pan=0.0, shutter=(0.0, 1.0), transform_times=(0.0, 1.0), **kw):
    """The Cornell box seen by an animated camera: over TransformTimes it moves `dolly` units towards the box and turns its view by
    `pan` degrees about the vertical axis (a rotation keyframe: slerp); `shutter` = (shutteropen, shutterclose).  Other keyword
    arguments go to cornell_box (materials, lights, textures, lensradius, sampler, integrator, ...)."""
    a = np.radians(pan)
    eye = [278.0, 273.0, -800.0 + dolly]
    look = [eye[0] + 800.0 * np.sin(a), 273.0, eye[2] + 800.0 * np.cos(a)]
    return cornell_box(xres=xres, yres=yres, spp=spp, camera_end=look_at_matrix(eye, look, [0, 1, 0]), shutter=shutter,
                       transform_times=transform_times, **kw)


def _set_integrator(h, integrator, maxdepth, strategy):
    """integrator: "path" | ("ao", nsamples, cossample) | ("direct", "all" | "one") | "whitted"."""
    if integrator == "path":
        h.integrator(maxdepth=maxdepth, lightsamplestrategy=strategy)
    elif integrator == "whitted":
        h.integrator_whitted(maxdepth=maxdepth)
    elif integrator[0] == "direct":
        h.integrator_direct(maxdepth=maxdepth, strategy=integrator[1])
    else:
        h.integrator_ao(nsamples=integrator[1], cossample=integrator[2])


def sky_map(width=64, height=32, seed=3):
    """Procedural lat-long radiance map (power-of-two resolution): blue-to-white gradient, a sun patch, noise."""
    rng = np.random.default_rng(seed)
    v = (np.arange(height) + 0.5) / height
    u = (np.arange(width) + 0.5) / width
    V, U = np.meshgrid(v, u, indexing="ij")
    up = np.cos(V * np.pi)  # +1 at the pole the map is wrapped around
    tex = np.stack([0.25 + 0.5 * (1 - up), 0.35 + 0.45 * (1 - up), 0.9 - 0.1 * up], -1) * np.where(up > 0, 1.0, 0.15)[..., None]
    sun = np.exp(-(((U - 0.3) * 2) ** 2 + (V - 0.2) ** 2) / 0.002)
    tex = tex + sun[..., None] * np.array([60.0, 50.0, 35.0])
    tex = tex * (0.9 + 0.2 * rng.random((height, width, 1)))
    return tex.astype(np.float32)


Y_UP = np.array([[1, 0, 0], [0, 0, 1], [0, -1, 0]], np.float32)  # light-space +z (the map's pole) -> world +y


def sky_scene(xres=64, yres=64, spp=16, maxdepth=5, strategy="spatial", env="constant", extra_lights=True, n_threads=8, sampler="sobol"):
    """Open scene under an InfiniteAreaLight: plastic floor, a matte, a mirror and a glass block, optionally an emissive quad and
    a point light.  `env`: "constant" (LightSource "infinite" without a map), "image" (sky_map, rotated so that its pole is +y),
    "two" (both: scene.infinite_lights holds two lights)."""
    h = HostScene()
    floor_m = h.material(_abi.MAT_PLASTIC, [0.4, 0.4, 0.4, 0.2, 0.2, 0.2, 0.1, 1.0])
    matte = h.material(_abi.MAT_MATTE, [0.6, 0.3, 0.2, 0.0])
    mirror = h.material(_abi.MAT_MIRROR, [0.9, 0.9, 0.9])
    glass = h.material(_abi.MAT_GLASS, [1, 1, 1, 1, 1, 1, 1.5, 0.0, 0.0, 1.0])
    if env in ("constant", "two"):
        h.light_infinite([0.6, 0.7, 0.9], scale=[1.5, 1.5, 1.5])
    h.trianglemesh(*_quad([-8, 0, -8], [-8, 0, 8], [8, 0, 8], [8, 0, -8]), material=floor_m)

    def block(x, z, sx, sz, hgt, rot, m):
        c, s_ = np.cos(rot), np.sin(rot)
        base = [[x + c * dx - s_ * dz, 0.0, z + s_ * dx + c * dz] for dx, dz in ((-sx, -sz), (-sx, sz), (sx, sz), (sx, -sz))]
        top = [[bx, hgt, bz] for bx, _, bz in base]
        h.trianglemesh(*_box(base, top), material=m)

    block(-2.2, 0.5, 0.9, 0.9, 1.8, 0.3, matte)
    if env in ("image", "two"):
        h.light_infinite([1.0, 1.0, 1.0], scale=[0.8, 0.8, 0.8], texels=sky_map(), light_to_world=Y_UP)
    block(0.2, 1.6, 0.8, 0.8, 2.6, -0.4, mirror)
    block(2.3, -0.3, 0.7, 0.7, 1.4, 0.6, glass)
    if extra_lights:
        h.trianglemesh(*_quad([-1, 4.0, -1], [1, 4.0, -1], [1, 4.0, 1], [-1, 4.0, 1]), material=matte, emit=[6.0, 5.0, 4.0])
        h.light_point([-3.0, 2.5, -2.0], [12.0, 12.0, 10.0])
    h.look_at([0.5, 3.0, -9.0], [0.0, 1.0, 0.0], [0, 1, 0])
    h.film(xres, yres)
    h.camera(fov=38.0)
    h.sampler(spp, name=sampler)
    h.integrator(maxdepth=maxdepth, lightsamplestrategy=strategy)
    h.world_end(n_threads=n_threads)
    return h


def landscape(xres=1920, yres=1080, spp=1024, maxdepth=5, n_trees=2000, grid=256, detail=12, seed=11, instancing="fixed", n_threads=8,
              strategy="spatial", sampler="sobol", integrator="path", n_prototypes=1, sky="map"):
    """Landscape stand-in (config C5): an fBm terrain, `n_trees` ObjectInstances of `n_prototypes` plant objects (tiers of cones of
    `detail` segments on a trunk; every prototype its own proportions, tier count and leaf material) with random rotation / non-uniform
    scale / position, a DistantLight sun and an InfiniteAreaLight sky (`sky`: "map" = a lat-long image, "constant").  BASELINE.json's
    configs[4] shape is n_trees = 3000, n_prototypes = 20 (SURVEY.md 8d item 4).
    `instancing`: "fixed" (pbrt-v3: instances are shaded) or "reference" (rs_pbrt's TransformedPrimitive: the path walks through
    them, quirk Q7)."""
    rng = np.random.default_rng(seed)
    h = HostScene()
    ground = h.material(_abi.MAT_MATTE, [0.35, 0.3, 0.2, 0.0])
    leaf = h.material(_abi.MAT_PLASTIC, [0.1, 0.35, 0.08, 0.05, 0.05, 0.05, 0.3, 1.0])
    bark = h.material(_abi.MAT_MATTE, [0.3, 0.2, 0.12, 20.0])
    h.light_infinite([1.0, 1.0, 1.0], scale=[0.6, 0.6, 0.6], texels=sky_map(128, 64, seed) if sky == "map" else None, light_to_world=Y_UP if sky == "map" else None)
    h.light_distant([0.4, 1.0, -0.3], [0.0, 0.0, 0.0], [3.0, 2.8, 2.4])
    # terrain
    u = np.linspace(0.0, 1.0, grid + 1)
    U, V = np.meshgrid(u, u, indexing="ij")
    H = 6.0 * _fbm(U * 3.0, V * 3.0, rng, octaves=5)
    P = np.stack([(U - 0.5) * 100.0, H, (V - 0.5) * 100.0], -1).reshape(-1, 3).astype(np.float32)
    i0 = (np.arange(grid)[:, None] * (grid + 1) + np.arange(grid)[None, :]).reshape(-1)
    idx = np.stack([i0, i0 + 1, i0 + grid + 2, i0, i0 + grid + 2, i0 + grid + 1], -1).reshape(-1).astype(np.uint32)
    h.trianglemesh(idx, P, material=ground)
    # the plant prototypes: ObjectBegin ... ObjectEnd each (api.rs:3001-3022)
    a = np.linspace(0.0, 2.0 * np.pi, detail, endpoint=False)
    ring = np.stack([np.cos(a), np.zeros_like(a), np.sin(a)], -1)
    protos = []
    prng = np.random.default_rng(seed + 101)
    for k in range(max(1, n_prototypes)):
        obj = h.object_begin()
        tiers = 1 if n_prototypes <= 1 else int(prng.integers(1, 4))
        radius = 1.2 if n_prototypes <= 1 else float(prng.uniform(0.8, 1.8))
        height = 4.0 if n_prototypes <= 1 else float(prng.uniform(3.0, 6.5))
        leaf_k = leaf if k == 0 else h.material(_abi.MAT_PLASTIC, [float(prng.uniform(0.05, 0.2)), float(prng.uniform(0.25, 0.45)), float(prng.uniform(0.04, 0.15)), 0.05, 0.05, 0.05,
                                                                     float(prng.uniform(0.2, 0.4)), 1.0])
        for t in range(tiers):
            y0 = 1.0 + (height - 1.0) * t / tiers * 0.8
            y1 = 1.0 + (height - 1.0) * (t + 1) / tiers
            r = radius * (1.0 - 0.25 * t)
            cone_p = np.concatenate([ring * r + [0, y0, 0], [[0.0, y1, 0.0]]]).astype(np.float32)
            cone_i = np.array([[j, (j + 1) % detail, detail] for j in range(detail)], np.uint32).reshape(-1)
            h.trianglemesh(cone_i, cone_p, material=leaf_k)
        trunk_p = np.concatenate([ring * 0.2, ring * 0.2 + [0, 1.0, 0]]).astype(np.float32)
        trunk_i = np.array([[j, (j + 1) % detail, detail + (j + 1) % detail, j, detail + (j + 1) % detail, detail + j] for j in range(detail)], np.uint32).reshape(-1)
        h.trianglemesh(trunk_i, trunk_p, material=bark)
        h.object_end()
        protos.append(obj)
    for i in range(n_trees):
        x, z = rng.uniform(-45.0, 45.0, 2)
        gi, gj = int((x / 100.0 + 0.5) * grid), int((z / 100.0 + 0.5) * grid)
        y = float(H[gi, gj]) - 0.05
        ang = rng.uniform(0.0, 2.0 * np.pi)
        sx, sy, sz = rng.uniform(0.6, 1.4), rng.uniform(0.7, 1.8), rng.uniform(0.6, 1.4)
        M = np.eye(4)
        M[:3, :3] = np.array([[np.cos(ang), 0, np.sin(ang)], [0, 1, 0], [-np.sin(ang), 0, np.cos(ang)]]) @ np.diag([sx, sy, sz])
        M[:3, 3] = [x, y, z]
        h.object_instance(protos[i % len(protos)], M.astype(np.float32))
    h.instancing(instancing)
    h.look_at([0.0, 14.0, -58.0], [0.0, 4.0, 0.0], [0, 1, 0])
    h.film(xres, yres)
    h.camera(fov=40.0)
    h.sampler(spp, name=sampler)
    _set_integrator(h, integrator, maxdepth, strategy)
    h.world_end(n_threads=n_threads)
    return h


def _fbm(u, v, rng, octaves=6):
    out = np.zeros_like(u)
    amp, freq = 1.0, 1.0
    for _ in range(octaves):
        a, b, c, d = rng.uniform(0.0, 2.0 * np.pi, 4)
        out += amp * (np.sin(freq * 2.0 * np.pi * u * 3.0 + a) * np.cos(freq * np.pi * v * 4.0 + b) +
                      0.5 * np.sin(freq * 2.0 * np.pi * (u * 5.0 + v * 2.0) + c) * np.sin(freq * np.pi * v * 7.0 + d))
        amp *= 0.5
        freq *= 2.0
    return out


def statue(n_side=1468, xres=1024, yres=1024, spp=128, maxdepth=5, seed=1234, with_normals=True, n_threads=8, crop=None, integrator="path",
           dolly=0.0):
    """Ganesha stand-in (config C3): an fBm-displaced, vertically stretched UV sphere of 2*n_side^2 triangles
    (n_side=1468 -> 4.31 M) with per-vertex normals, on a ground quad, lit by 3 rectangular area lights
    (6 light triangles); matte statue + plastic ground.  `dolly` != 0: the camera moves that far towards the statue over the
    shutter interval (motion blur)."""
    rng = np.random.default_rng(seed)
    h = HostScene()
    body = h.material(_abi.MAT_MATTE, [0.62, 0.47, 0.33, 0.0])
    ground = h.material(_abi.MAT_PLASTIC, [0.35, 0.35, 0.38, 0.25, 0.25, 0.25, 0.1, 1.0])
    lm = h.material(_abi.MAT_MATTE, [0.5, 0.5, 0.5, 0.0])
    nu, nv = n_side, n_side
    u = np.linspace(0.0, 1.0, nu + 1, dtype=np.float64)
    v = np.linspace(0.0, 1.0, nv + 1, dtype=np.float64)
    uu, vv = np.meshgrid(u, v, indexing="xy")
    theta = vv * np.pi
    phi = uu * 2.0 * np.pi
    # periodic in u so the seam closes
    r = 1.0 + 0.12 * _fbm(uu, vv, rng) * np.sin(theta) ** 2 + 0.25 * np.sin(theta * 3.0) ** 2
    x = r * np.sin(theta) * np.cos(phi)
    y = 1.6 * r * np.cos(theta) + 1.9
    z = r * np.sin(theta) * np.sin(phi)
    P = np.stack([x, y, z], -1).astype(np.float32).reshape(-1, 3)
    # finite-difference normals
    Pg = P.reshape(nv + 1, nu + 1, 3).astype(np.float64)
    du = np.roll(Pg, -1, 1) - np.roll(Pg, 1, 1)
    dv = np.empty_like(Pg)
    dv[1:-1] = Pg[2:] - Pg[:-2]
    dv[0] = Pg[1] - Pg[0]
    dv[-1] = Pg[-1] - Pg[-2]
    N = np.cross(dv, du)
    ln = np.linalg.norm(N, axis=-1, keepdims=True)
    N = np.where(ln > 0, N / np.maximum(ln, 1e-30), np.array([0.0, 1.0, 0.0]))
    N = N.astype(np.float32).reshape(-1, 3)
    i = np.arange(nu, dtype=np.uint32)[None, :]
    j = np.arange(nv, dtype=np.uint32)[:, None]
    a = j * (nu + 1) + i
    b = a + 1
    c = a + (nu + 1)
    d = c + 1
    idx = np.stack([a, c, b, b, c, d], -1).astype(np.uint32).reshape(-1)
    h.trianglemesh(idx, P, N=N if with_normals else None, material=body)
    G = 12.0
    h.trianglemesh(*_quad([-G, 0, -G], [-G, 0, G], [G, 0, G], [G, 0, -G]), material=ground)
    for (cx, cy, cz, sx, sz, L) in [(-3.0, 7.0, -2.0, 1.5, 1.0, [40, 36, 30]), (3.5, 6.0, 1.0, 1.0, 1.5, [18, 22, 30]), (0.0, 8.0, 4.0, 2.0, 0.8, [25, 25, 25])]:
        h.trianglemesh(*_quad([cx - sx, cy, cz - sz], [cx + sx, cy, cz - sz], [cx + sx, cy, cz + sz], [cx - sx, cy, cz + sz]), material=lm,
                       emit=[float(t) for t in L])
    h.look_at([0.0, 3.2, -7.5], [0.0, 2.0, 0.0], [0, 1, 0])
    if dolly:
        eye = np.array([0.0, 3.2, -7.5]) + dolly * np.array([0.0, -1.2, 7.5]) / np.linalg.norm([0.0, -1.2, 7.5])
        _camera_motion(h, look_at_matrix(eye, [0.0, 2.0, 0.0], [0, 1, 0]), (0.0, 1.0))
    h.film(xres, yres, crop=crop)
    h.camera(fov=38.0)
    h.sampler(spp)
    _set_integrator(h, integrator, maxdepth, "spatial")
    h.world_end(n_threads=n_threads)
    return h


def conference(xres=1280, yres=720, spp=512, maxdepth=5, seed=7, n_chairs=40, detail=24, n_light_quads=64, n_threads=8, crop=None):
    """Conference-room stand-in (config C4): room, table, `n_chairs` chairs made of tessellated boxes
    (instanced by COPY), 7 material kinds, n_light_quads ceiling light quads (2 area lights each)."""
    rng = np.random.default_rng(seed)
    h = HostScene()
    mats = {
        "wall": h.material(_abi.MAT_MATTE, [0.7, 0.68, 0.62, 20.0]),  # Oren-Nayar
        "floor": h.material(_abi.MAT_SUBSTRATE, [0.35, 0.2, 0.12, 0.08, 0.08, 0.08, 0.08, 0.12, 1.0]),
        "table": h.material(_abi.MAT_PLASTIC, [0.3, 0.15, 0.08, 0.4, 0.4, 0.4, 0.05, 1.0]),
        "chair": h.material(_abi.MAT_UBER, [0.1, 0.12, 0.3, 0.2, 0.2, 0.2, 0.05, 0.05, 0.05, 0, 0, 0, 1, 1, 1, 0.1, 0.1, 1.5, 1.0]),
        "metal": h.material(_abi.MAT_METAL, [0.2, 0.92, 1.1, 3.9, 2.45, 2.14, 0.02, 0.02, 1.0]),
        "mirror": h.material(_abi.MAT_MIRROR, [0.9, 0.9, 0.9]),
        "glass": h.material(_abi.MAT_GLASS, [1, 1, 1, 1, 1, 1, 1.5, 0.0, 0.0, 1.0]),
        "light": h.material(_abi.MAT_MATTE, [0.6, 0.6, 0.6, 0.0]),
    }

    def tess_box(lo, hi, n):
        """Axis-aligned box with each face split into n x n quads."""
        lo = np.asarray(lo, np.float64)
        hi = np.asarray(hi, np.float64)
        Ps, Is, base = [], [], 0
        t = np.linspace(0.0, 1.0, n + 1)
        for axis in range(3):
            for side in (0, 1):
                a1, a2 = [k for k in range(3) if k != axis]
                g1, g2 = np.meshgrid(t, t, indexing="xy")
                pts = np.zeros((n + 1, n + 1, 3))
                pts[..., axis] = hi[axis] if side else lo[axis]
                pts[..., a1] = lo[a1] + g1 * (hi[a1] - lo[a1])
                pts[..., a2] = lo[a2] + g2 * (hi[a2] - lo[a2])
                ii = np.arange(n)[None, :]
                jj = np.arange(n)[:, None]
                a = jj * (n + 1) + ii
                q = np.stack([a, a + 1, a + n + 2, a, a + n + 2, a + n + 1], -1).reshape(-1) + base
                Ps.append(pts.reshape(-1, 3))
                Is.append(q)
                base += (n + 1) * (n + 1)
        return np.concatenate(Is).astype(np.uint32), np.concatenate(Ps).astype(np.float32)

    X, Y, Z = 12.0, 4.0, 8.0
    h.trianglemesh(*tess_box([-X, -0.1, -Z], [X, 0.0, Z], 8), material=mats["floor"])
    h.trianglemesh(*tess_box([-X, Y, -Z], [X, Y + 0.1, Z], 8), material=mats["wall"])
    h.trianglemesh(*tess_box([-X - 0.1, 0, -Z], [-X, Y, Z], 8), material=mats["wall"])
    h.trianglemesh(*tess_box([X, 0, -Z], [X + 0.1, Y, Z], 8), material=mats["wall"])
    h.trianglemesh(*tess_box([-X, 0, Z], [X, Y, Z + 0.1], 8), material=mats["wall"])
    h.trianglemesh(*tess_box([-X, 0, -Z - 0.1], [X, Y, -Z], 8), material=mats["wall"])
    h.trianglemesh(*tess_box([-6.0, 1.0, -1.6], [6.0, 1.12, 1.6], detail), material=mats["table"])
    for lx in (-5.5, 5.5):
        for lz in (-1.3, 1.3):
            h.trianglemesh(*tess_box([lx - 0.1, 0, lz - 0.1], [lx + 0.1, 1.0, lz + 0.1], 4), material=mats["metal"])
    h.trianglemesh(*tess_box([-3.0, 1.2, X * 0 + Z - 0.05], [3.0, 3.2, Z - 0.02], 4), material=mats["mirror"])
    h.trianglemesh(*tess_box([-0.4, 1.12, -0.4], [0.4, 1.9, 0.4], 6), material=mats["glass"])
    per_side = max(1, n_chairs // 2)
    for k in range(n_chairs):
        side = -1.0 if k < per_side else 1.0
        cx = -5.5 + 11.0 * ((k % per_side) + 0.5) / per_side + float(rng.uniform(-0.05, 0.05))
        cz = side * 2.6
        h.trianglemesh(*tess_box([cx - 0.3, 0.55, cz - 0.3], [cx + 0.3, 0.65, cz + 0.3], detail // 2), material=mats["chair"])
        h.trianglemesh(*tess_box([cx - 0.3, 0.65, cz + side * 0.25], [cx + 0.3, 1.4, cz + side * 0.3], detail // 2), material=mats["chair"])
        for dx in (-0.25, 0.25):
            for dz in (-0.25, 0.25):
                h.trianglemesh(*tess_box([cx + dx - 0.03, 0, cz + dz - 0.03], [cx + dx + 0.03, 0.55, cz + dz + 0.03], 2), material=mats["metal"])
    nlx = int(np.ceil(np.sqrt(n_light_quads * 1.5)))
    nlz = int(np.ceil(n_light_quads / nlx))
    made = 0
    for a in range(nlx):
        for b in range(nlz):
            if made >= n_light_quads:
                break
            cx = -X + 2 * X * (a + 0.5) / nlx
            cz = -Z + 2 * Z * (b + 0.5) / nlz
            yq = Y - 0.01
            h.trianglemesh(*_quad([cx - 0.4, yq, cz - 0.25], [cx + 0.4, yq, cz - 0.25], [cx + 0.4, yq, cz + 0.25], [cx - 0.4, yq, cz + 0.25]),
                           material=mats["light"], emit=[9.0, 9.0, 8.5])
            made += 1
    h.look_at([-10.5, 2.4, -6.5], [0.0, 1.2, 0.5], [0, 1, 0])
    h.film(xres, yres, crop=crop)
    h.camera(fov=55.0)
    h.sampler(spp)
    h.integrator(maxdepth=maxdepth)
    h.world_end(n_threads=n_threads)
    return h


def mapped_walls(xres=64, yres=64, spp=8):
    """Three walls with image textures under the spherical, cylindrical and planar TextureMapping2D kinds (texture.rs:123-252), one of
    them bump-mapped through a planar mapping; a point light and a dim sky."""
    rng = np.random.default_rng(51)
    h = HostScene()
    c, s = np.cos(0.4), np.sin(0.4)
    w2t = np.array([[c, 0, s, -0.3], [0, 1, 0, -1.0], [-s, 0, c, 0.2], [0, 0, 0, 1]], np.float32)
    t_sph = h.texture_mapping(h.texture_image((0.1 + 0.8 * rng.random((16, 32, 3))).astype(np.float32)), "spherical", w2t)
    t_cyl = h.texture_mapping(h.texture_image((0.1 + 0.8 * rng.random((16, 16, 3))).astype(np.float32), trilinear=True), "cylindrical", w2t)
    t_pla = h.texture_mapping(h.texture_image((0.1 + 0.8 * rng.random((8, 8, 3))).astype(np.float32), udelta=0.25, vdelta=-0.5), "planar",
                              [0.3, 0.0, 0.1, 0.0, 0.2, 0.25])
    t_bmp = h.texture_mapping(h.texture_image(rng.random((16, 16, 3)).astype(np.float32), float_valued=True, scale=0.5), "planar", [0.5, 0, 0, 0, 0, 0.5])
    m_sph = h.material(_abi.MAT_MATTE, [0.5, 0.5, 0.5, 0.0], textures={0: t_sph})
    m_cyl = h.material(_abi.MAT_PLASTIC, [0.5, 0.5, 0.5, 0.2, 0.2, 0.2, 0.2, 1.0], textures={0: t_cyl}, bump=t_bmp)
    m_pla = h.material(_abi.MAT_MATTE, [0.5, 0.5, 0.5, 10.0], textures={0: t_pla})
    h.light_infinite([1.0, 1.0, 1.0], scale=[0.6, 0.6, 0.6])
    h.light_point([0.0, 4.0, -2.0], [25.0, 25.0, 25.0])
    quad = np.array([0, 1, 2, 0, 2, 3], np.uint32)
    h.trianglemesh(quad, np.array([[-5, 0, -5], [5, 0, -5], [5, 0, 5], [-5, 0, 5]], np.float32), material=m_pla)
    h.trianglemesh(quad, np.array([[-3, 0, 3], [3, 0, 3], [3, 4, 3], [-3, 4, 3]], np.float32), material=m_sph)
    h.trianglemesh(quad, np.array([[-3, 0, -2], [-3, 0, 3], [-3, 4, 3], [-3, 4, -2]], np.float32), material=m_cyl)
    h.look_at([1.5, 2.5, -6.0], [0.0, 1.0, 1.0], [0, 1, 0])
    h.film(xres, yres)
    h.camera(fov=45.0)
    h.sampler(spp)
    h.integrator(maxdepth=3, lightsamplestrategy="uniform")
    h.world_end(n_threads=1)
    return h
