"""Float64 restatement of the surface-scattering mathematics, written from the formulas of pbrt-v3 (Pharr, Jakob, Humphreys,
"Physically Based Rendering", 3rd ed.: chapter 8 for the BxDFs and Fresnel terms, chapter 14 for the light transport) -- not from
the CUDA kernels and not from oracle/.  It is the second reference of tests/test_gpu_closed_forms.py: the kernels are held to plain
mathematics here, and to the oracle elsewhere.

Where rs_pbrt departs from pbrt-v3 this module follows rs_pbrt and says where:
  * plastic's specular Fresnel term is FresnelDielectric(eta_i = 1.5, eta_t = 1.0) (src/materials/plastic.rs:99-102);
  * TrowbridgeReitzDistribution::new clamps both alphas to >= 0.001 (src/core/microfacet.rs:232-238);
  * a MixMaterial scales every lobe of its first child by clamp(amount) and of its second child by clamp(1 - that); a child that is
    itself a mix ignores the scale handed down (src/materials/mixmat.rs:41-98, the unused `_scale` at :48);
  * the specular lobes report a cosine pdf (src/core/reflection.rs:828-834) and a scaled non-specular lobe's sample_f scales f twice
    (reflection.rs:982-983).  Neither changes a value computed here: f of a specular lobe is 0 for every pair of directions, next-event
    estimation never asks a specular lobe for its pdf, and Bsdf::sample_f recomputes f of a non-specular sample (reflection.rs:393-410).
Everything works on NumPy float64 arrays; directions are (..., 3) arrays, in the local shading frame (z = shading normal) unless a
function says otherwise, and spectra are (..., 3) RGB arrays."""
import math

import numpy as np

# material kinds and their params[] layouts, as include/pbrt_gpu.h numbers them
MATTE, PLASTIC, METAL, MIRROR, GLASS, UBER, SUBSTRATE, TRANSLUCENT, MIX = range(9)

REFLECTION, TRANSMISSION = 1, 2


def _dot(a, b):
    return np.sum(a * b, axis=-1)


def _normalize(v):
    return v / np.linalg.norm(v, axis=-1, keepdims=True)


# ---- Fresnel (section 8.2) ----------------------------------------------------------------------------------------------------

def fr_dielectric(cos_i, eta_i, eta_t):
    """Unpolarised Fresnel reflectance of a dielectric interface (eq. 8.4-8.5).  cos_i < 0: the ray arrives from the eta_t side."""
    cos_i = np.clip(np.asarray(cos_i, np.float64), -1.0, 1.0)
    inside = cos_i < 0.0
    ei = np.where(inside, eta_t, eta_i)
    et = np.where(inside, eta_i, eta_t)
    ci = np.abs(cos_i)
    sin_t = ei / et * np.sqrt(np.maximum(0.0, 1.0 - ci * ci))
    tir = sin_t >= 1.0
    ct = np.sqrt(np.maximum(0.0, 1.0 - sin_t * sin_t))
    r_par = (et * ci - ei * ct) / (et * ci + ei * ct)
    r_perp = (ei * ci - et * ct) / (ei * ci + et * ct)
    return np.where(tir, 1.0, 0.5 * (r_par ** 2 + r_perp ** 2))


def fr_conductor(cos_i, eta, k):
    """Fresnel reflectance of a conductor with complex index n = eta + i k against vacuum, for unpolarised light: the complex
    amplitudes r_s = (cos_i - n cos_t) / (cos_i + n cos_t), r_p = (n cos_i - cos_t) / (n cos_i + cos_t) with Snell's law in complex
    form, n cos_t = sqrt(n^2 - sin_i^2).  (pbrt-v3 eq. 8.6 is the same quantity written in real arithmetic.)  Spectra in, spectra out."""
    c = np.clip(np.asarray(cos_i, np.float64), -1.0, 1.0)[..., None]
    n = np.asarray(eta, np.float64) + 1j * np.asarray(k, np.float64)
    s2 = 1.0 - c * c
    n_cos_t = np.sqrt(n * n - s2)
    rs = (c - n_cos_t) / (c + n_cos_t)
    rp = (n * n * c - n_cos_t) / (n * n * c + n_cos_t)
    return 0.5 * (np.abs(rs) ** 2 + np.abs(rp) ** 2)


def schlick(rs, cos):
    return rs + (1.0 - rs) * (1.0 - cos[..., None]) ** 5


# ---- Trowbridge-Reitz (GGX) microfacets (section 8.4) ------------------------------------------------------------------------

def roughness_to_alpha(roughness):
    """The "remaproughness" polynomial in x = ln(roughness), roughness clamped to >= 1e-3 (src/core/microfacet.rs:243-255)."""
    x = math.log(max(float(roughness), 1e-3))
    return 1.62142 + 0.819955 * x + 0.1734 * x ** 2 + 0.0171201 * x ** 3 + 0.000640711 * x ** 4


def _tan2_cos2phi_sin2phi(w):
    s2 = np.maximum(0.0, 1.0 - w[..., 2] ** 2)
    rho2 = w[..., 0] ** 2 + w[..., 1] ** 2
    with np.errstate(invalid="ignore", divide="ignore"):
        c2 = np.where(rho2 > 0.0, w[..., 0] ** 2 / np.where(rho2 > 0.0, rho2, 1.0), 1.0)
        t2 = s2 / (w[..., 2] ** 2)
    return t2, c2, 1.0 - c2


def tr_d(wh, ax, ay):
    """D(wh) = 1 / (pi ax ay cos^4 th (1 + tan^2 th (cos^2 ph / ax^2 + sin^2 ph / ay^2))^2)  (eq. 8.11, anisotropic)."""
    t2, c2, s2 = _tan2_cos2phi_sin2phi(wh)
    e = t2 * (c2 / ax ** 2 + s2 / ay ** 2)
    cos4 = wh[..., 2] ** 4
    with np.errstate(invalid="ignore", divide="ignore"):
        d = 1.0 / (math.pi * ax * ay * cos4 * (1.0 + e) ** 2)
    return np.where(np.isfinite(t2), d, 0.0)


def tr_lambda(w, ax, ay):
    """Smith's Lambda(w) = (-1 + sqrt(1 + alpha^2 tan^2 th)) / 2 with alpha^2 = cos^2 ph ax^2 + sin^2 ph ay^2 (eq. 8.13, 8.14)."""
    t2, c2, s2 = _tan2_cos2phi_sin2phi(w)
    a2 = c2 * ax ** 2 + s2 * ay ** 2
    return np.where(np.isfinite(t2), 0.5 * (np.sqrt(1.0 + a2 * np.where(np.isfinite(t2), t2, 0.0)) - 1.0), 0.0)


def tr_g1(w, ax, ay):
    return 1.0 / (1.0 + tr_lambda(w, ax, ay))


def tr_g(wo, wi, ax, ay):
    """Height-correlated masking-shadowing G = 1 / (1 + Lambda(wo) + Lambda(wi)) (eq. 8.12)."""
    return 1.0 / (1.0 + tr_lambda(wo, ax, ay) + tr_lambda(wi, ax, ay))


# ---- lobes -----------------------------------------------------------------------------------------------------------------
# A lobe is a dict: kind, side (REFLECTION / TRANSMISSION), scale (the MixMaterial's spectrum, or ones) and its own parameters.
# Specular lobes are listed with kind "specular" and contribute nothing to f.

def _lobe(kind, side, **kw):
    d = dict(kind=kind, side=side, scale=np.ones(3))
    d.update({k: (np.asarray(v, np.float64) if isinstance(v, (list, tuple, np.ndarray)) else v) for k, v in kw.items()})
    return d


def lobe_f(L, wo, wi):
    """f(wo, wi) of one lobe, in the local frame; wo, wi (..., 3) unit vectors."""
    k = L["kind"]
    shape = np.broadcast_shapes(wo.shape, wi.shape)[:-1] + (3,)
    co, ci = wo[..., 2], wi[..., 2]
    if k == "specular":
        return np.zeros(shape)
    if k == "lambert":  # eq. 8.9: R / pi
        return np.broadcast_to(L["scale"] * L["R"] / math.pi, shape).copy()
    if k == "lambert_t":  # LambertianTransmission: T / pi (reflection.rs:1010-1016)
        return np.broadcast_to(L["scale"] * L["T"] / math.pi, shape).copy()
    if k == "oren_nayar":  # eq. 8.10 with A, B of section 8.4.2; alpha = max(th_i, th_o), beta = min(th_i, th_o)
        sin_i = np.sqrt(np.maximum(0.0, 1.0 - ci ** 2))
        sin_o = np.sqrt(np.maximum(0.0, 1.0 - co ** 2))
        both = (sin_i > 1e-4) & (sin_o > 1e-4)
        with np.errstate(invalid="ignore", divide="ignore"):
            cos_dphi = (wi[..., 0] * wo[..., 0] + wi[..., 1] * wo[..., 1]) / (sin_i * sin_o)
        max_cos = np.where(both, np.maximum(np.nan_to_num(cos_dphi), 0.0), 0.0)
        i_steeper = np.abs(ci) > np.abs(co)
        sin_alpha = np.where(i_steeper, sin_o, sin_i)
        tan_beta = np.where(i_steeper, sin_i / np.abs(ci), sin_o / np.abs(co))
        return L["scale"] * L["R"] / math.pi * (L["A"] + L["B"] * max_cos * sin_alpha * tan_beta)[..., None]
    if k == "mf_refl":  # Torrance-Sparrow, eq. 8.18: R D G F / (4 |cos_i| |cos_o|), F at the microfacet angle wi.wh
        wh = wi + wo
        zero = (co == 0.0) | (ci == 0.0) | np.all(wh == 0.0, axis=-1)
        wh = _normalize(np.where(zero[..., None], np.array([0.0, 0.0, 1.0]), wh))
        c = _dot(wi, wh)
        if L["fresnel"] == "conductor":
            F = fr_conductor(c, L["eta"], L["k"])
        else:
            F = fr_dielectric(c, L["eta_i"], L["eta_t"])[..., None] * np.ones(3)
        ax, ay = L["ax"], L["ay"]
        v = (tr_d(wh, ax, ay) * tr_g(wo, wi, ax, ay) / (4.0 * np.abs(ci) * np.abs(co)))[..., None] * F * L["R"] * L["scale"]
        return np.where(zero[..., None], 0.0, v)
    if k == "mf_trans":  # eq. 8.20 for radiance: the eta^2 of the half-vector Jacobian cancels against the 1 / eta^2 of radiance
        eta = np.where(co > 0.0, L["eta_b"] / L["eta_a"], L["eta_a"] / L["eta_b"])
        wh = _normalize(wo + wi * eta[..., None])
        wh = np.where((wh[..., 2] < 0.0)[..., None], -wh, wh)
        ow, iw = _dot(wo, wh), _dot(wi, wh)
        bad = (co * ci >= 0.0) | (ow * iw > 0.0)
        F = fr_dielectric(ow, L["eta_a"], L["eta_b"])
        ax, ay = L["ax"], L["ay"]
        with np.errstate(invalid="ignore", divide="ignore"):
            v = np.abs(tr_d(wh, ax, ay) * tr_g(wo, wi, ax, ay) * np.abs(iw) * np.abs(ow) / (ci * co * (ow + eta * iw) ** 2))
        return np.where(bad[..., None], 0.0, ((1.0 - F) * v)[..., None] * L["T"] * L["scale"])
    if k == "fresnel_blend":  # Ashikhmin-Shirley, eq. 8.22 (diffuse) and 8.23 (glossy, Schlick's Fresnel at wi.wh)
        rd, rs = L["Rd"], L["Rs"]
        diffuse = (28.0 / (23.0 * math.pi)) * rd * (1.0 - rs) * ((1.0 - (1.0 - 0.5 * np.abs(ci)) ** 5) * (1.0 - (1.0 - 0.5 * np.abs(co)) ** 5))[..., None]
        wh = wi + wo
        zero = np.all(wh == 0.0, axis=-1)
        wh = _normalize(np.where(zero[..., None], np.array([0.0, 0.0, 1.0]), wh))
        c = _dot(wi, wh)
        spec = schlick(rs, c) * (tr_d(wh, L["ax"], L["ay"]) / (4.0 * np.abs(c) * np.maximum(np.abs(ci), np.abs(co))))[..., None]
        return np.where(zero[..., None], 0.0, L["scale"] * (diffuse + spec))
    raise ValueError(k)


def bsdf_f_local(lobes, wo, wi, reflect=None):
    """Bsdf::f over the non-specular lobes (section 9.1): the reflection lobes where wi and wo lie on the same side of the geometric
    surface, the transmission lobes where they do not.  `reflect` (bool array) decides the side; by default the local z does."""
    wo, wi = np.broadcast_arrays(np.asarray(wo, np.float64), np.asarray(wi, np.float64))
    if reflect is None:
        reflect = wo[..., 2] * wi[..., 2] > 0.0
    out = np.zeros(wo.shape[:-1] + (3,))
    for L in lobes:
        on_side = reflect if L["side"] == REFLECTION else ~reflect
        out += np.where(on_side[..., None], lobe_f(L, wo, wi), 0.0)
    return np.where((wo[..., 2] == 0.0)[..., None], 0.0, out)


def bsdf_f_world(lobes, ns, ss, ng, wo_w, wi_w):
    """Bsdf::f with world directions: frame (ss, ns x ss, ns), geometric normal ng for the reflect / transmit choice."""
    ns, ss, ng = (np.asarray(v, np.float64) for v in (ns, ss, ng))
    ts = np.cross(ns, ss)
    loc = lambda w: np.stack([_dot(w, ss), _dot(w, ts), _dot(w, ns)], -1)
    reflect = _dot(wi_w, ng) * _dot(wo_w, ng) > 0.0
    return bsdf_f_local(lobes, loc(wo_w), loc(wi_w), reflect)


# ---- materials (chapter 9: how each material assembles its lobes) ----------------------------------------------------------

def _alphas(u, v, remap):
    if remap:
        u, v = roughness_to_alpha(u), roughness_to_alpha(v)
    return max(u, 0.001), max(v, 0.001)


def material_lobes(materials, index):
    """The lobes of material `index` of a list of (kind, params) pairs (params as in include/pbrt_gpu.h); a MIX names earlier
    entries of the same list."""
    kind, p = materials[index]
    p = np.zeros(24) + np.pad(np.asarray(p, np.float64), (0, 24 - len(p)))
    pos = lambda i: np.maximum(p[i:i + 3], 0.0)
    black = lambda s: not np.any(s > 0.0)
    out = []
    if kind == MATTE:
        sigma = min(max(p[3], 0.0), 90.0)
        if not black(pos(0)):
            if sigma == 0.0:
                out.append(_lobe("lambert", REFLECTION, R=pos(0)))
            else:
                s2 = math.radians(sigma) ** 2
                out.append(_lobe("oren_nayar", REFLECTION, R=pos(0), A=1.0 - s2 / (2.0 * (s2 + 0.33)), B=0.45 * s2 / (s2 + 0.09)))
    elif kind == PLASTIC:
        if not black(pos(0)):
            out.append(_lobe("lambert", REFLECTION, R=pos(0)))
        if not black(pos(3)):
            a, _ = _alphas(p[6], p[6], p[7] != 0.0)
            out.append(_lobe("mf_refl", REFLECTION, R=pos(3), ax=a, ay=a, fresnel="dielectric", eta_i=1.5, eta_t=1.0))  # plastic.rs:99-102
    elif kind == METAL:
        ax, ay = _alphas(p[6], p[7], p[8] != 0.0)
        out.append(_lobe("mf_refl", REFLECTION, R=np.ones(3), ax=ax, ay=ay, fresnel="conductor", eta=p[0:3], k=p[3:6]))
    elif kind == MIRROR:
        out.append(_lobe("specular", REFLECTION))
    elif kind == GLASS:
        if p[7] == 0.0 and p[8] == 0.0:
            out.append(_lobe("specular", REFLECTION))
            out.append(_lobe("specular", TRANSMISSION))
        else:
            ax, ay = _alphas(p[7], p[8], p[9] != 0.0)
            if not black(pos(0)):
                out.append(_lobe("mf_refl", REFLECTION, R=pos(0), ax=ax, ay=ay, fresnel="dielectric", eta_i=1.0, eta_t=p[6]))
            if not black(pos(3)):
                out.append(_lobe("mf_trans", TRANSMISSION, T=pos(3), ax=ax, ay=ay, eta_a=1.0, eta_b=p[6]))
    elif kind == UBER:
        op = pos(12)
        if not black(np.maximum(1.0 - op, 0.0)):
            out.append(_lobe("specular", TRANSMISSION))  # the pass-through of an opacity below 1
        if not black(op * pos(0)):
            out.append(_lobe("lambert", REFLECTION, R=op * pos(0)))
        if not black(op * pos(3)):
            ax, ay = _alphas(p[15], p[16], p[18] != 0.0)
            out.append(_lobe("mf_refl", REFLECTION, R=op * pos(3), ax=ax, ay=ay, fresnel="dielectric", eta_i=1.0, eta_t=p[17]))
        if not black(op * pos(6)):
            out.append(_lobe("specular", REFLECTION))
        if not black(op * pos(9)):
            out.append(_lobe("specular", TRANSMISSION))
    elif kind == SUBSTRATE:
        if not (black(pos(0)) and black(pos(3))):
            ax, ay = _alphas(p[6], p[7], p[8] != 0.0)
            out.append(_lobe("fresnel_blend", REFLECTION, Rd=pos(0), Rs=pos(3), ax=ax, ay=ay))
    elif kind == TRANSLUCENT:  # eta 1.5, radiance transport
        kd, ks, r, t = pos(0), pos(3), pos(6), pos(9)
        if not (black(r) and black(t)):
            if not black(kd):
                if not black(r):
                    out.append(_lobe("lambert", REFLECTION, R=r * kd))
                if not black(t):
                    out.append(_lobe("lambert_t", TRANSMISSION, T=t * kd))
            if not black(ks):
                a, _ = _alphas(p[12], p[12], p[13] != 0.0)
                if not black(r):
                    out.append(_lobe("mf_refl", REFLECTION, R=r * ks, ax=a, ay=a, fresnel="dielectric", eta_i=1.0, eta_t=1.5))
                if not black(t):
                    out.append(_lobe("mf_trans", TRANSMISSION, T=t * ks, ax=a, ay=a, eta_a=1.0, eta_b=1.5))
    elif kind == MIX:
        s1 = np.clip(p[0:3], 0.0, 1.0)
        s2 = np.clip(1.0 - s1, 0.0, 1.0)
        for child, s in ((int(p[3]), s1), (int(p[4]), s2)):
            lobes = material_lobes(materials, child)
            if materials[child][0] != MIX:  # a nested mix keeps its own scales (mixmat.rs:48)
                for L in lobes:
                    L["scale"] = s
            out += lobes
    else:
        raise ValueError(kind)
    return out


# ---- area lights (section 14.2 / Lambert's formula) ------------------------------------------------------------------------

def clip_polygon(verts, p, n):
    """The part of the polygon `verts` (m, 3) on the side n.(x - p) >= 0 (Sutherland-Hodgman against one plane)."""
    out = []
    m = len(verts)
    for i in range(m):
        a, b = verts[i], verts[(i + 1) % m]
        da, db = float(np.dot(n, a - p)), float(np.dot(n, b - p))
        if da >= 0.0:
            out.append(a)
        if (da >= 0.0) != (db >= 0.0):
            out.append(a + (b - a) * (da / (da - db)))
    return np.array(out, np.float64).reshape(-1, 3)


def polygon_form_factor(p, n, verts):
    """Projected solid angle  Phi = integral over the polygon of max(cos th, 0) d omega  seen from p with normal n (Lambert's polygon
    formula: Phi = 1/2 |sum_i gamma_i n . (u_i x u_i+1) / |u_i x u_i+1||, u_i the unit vectors to the vertices, gamma_i the angle
    between consecutive ones).  The polygon is clipped to the upper half-space of (p, n) first.  The irradiance at p from a
    uniform emitter of radiance Le is Le * Phi; a Lambertian surface of reflectance Kd there reflects Kd / pi * Le * Phi."""
    p, n = np.asarray(p, np.float64), np.asarray(n, np.float64)
    v = clip_polygon(np.asarray(verts, np.float64), p, n)
    if len(v) < 3:
        return 0.0
    u = _normalize(v - p)
    acc = 0.0
    for i in range(len(u)):
        a, b = u[i], u[(i + 1) % len(u)]
        c = np.cross(a, b)
        s = np.linalg.norm(c)
        if s > 0.0:
            acc += math.atan2(s, float(np.dot(a, b))) * float(np.dot(n, c)) / s
    return abs(0.5 * acc)


# ---- directional albedo by quadrature --------------------------------------------------------------------------------------

def _gauss_panels(a, b, panels, order):
    x, w = np.polynomial.legendre.leggauss(order)
    edges = np.linspace(a, b, panels + 1)
    h = np.diff(edges)[:, None]
    return ((edges[:-1, None] + h * (x + 1.0) / 2.0).ravel(), (h * w / 2.0).ravel())


def _albedo_at(lobes, wo, panels, n_phi, order=8):
    """rho(wo) with mu = cos th_i in composite Gauss-Legendre panels and phi on the periodic trapezoid rule (d omega = d mu d phi).
    Panel edges sit where the integrand jumps: the horizon mu = 0 (the reflect / transmit switch), and for a microfacet transmission
    lobe the circle where the generalised half vector wo + eta wi crosses the horizon, mu = -cos th_o / eta: there it is flipped
    and the Fresnel term F(wo . wh) changes sides of the interface."""
    acc = np.zeros(3)
    phi = (np.arange(n_phi) + 0.5) * (2.0 * math.pi / n_phi)
    cp, sp = np.cos(phi), np.sin(phi)
    edges = {-1.0, 0.0, 1.0}
    for L in lobes:
        if L["kind"] == "mf_trans" and wo[2] != 0.0:
            eta = L["eta_b"] / L["eta_a"] if wo[2] > 0.0 else L["eta_a"] / L["eta_b"]
            if abs(wo[2] / eta) < 1.0:
                edges.add(-wo[2] / eta)
    edges = sorted(edges)
    for a, b in zip(edges[:-1], edges[1:]):
        mu, w = _gauss_panels(a, b, max(1, int(math.ceil(panels * (b - a)))), order)
        st = np.sqrt(np.maximum(0.0, 1.0 - mu * mu))
        wi = np.stack([st[:, None] * cp[None, :], st[:, None] * sp[None, :], np.broadcast_to(mu[:, None], (mu.size, n_phi))], -1)
        f = bsdf_f_local(lobes, np.asarray(wo, np.float64)[None, None, :], wi)
        acc += np.einsum("ijc,i->c", f * np.abs(mu)[:, None, None], w) * (2.0 * math.pi / n_phi)
    return acc


def albedo(lobes, wo, panels=48, n_phi=768, rtol=1e-6):
    """Directional albedo rho(wo) = integral over the sphere of f(wo, wi) |cos th_i| d omega_i, RGB, wo in the local frame.  Evaluated
    at two resolutions (the second with twice the panels and twice the phi nodes); asserts that they agree to `rtol`."""
    wo = np.asarray(wo, np.float64)
    lo = _albedo_at(lobes, wo, panels, n_phi)
    hi = _albedo_at(lobes, wo, 2 * panels, 2 * n_phi)
    scale = max(float(np.max(np.abs(hi))), 1e-300)
    assert np.all(np.abs(hi - lo) <= rtol * scale), ("albedo quadrature not converged", lo, hi)
    return hi
