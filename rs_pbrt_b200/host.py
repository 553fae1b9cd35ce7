"""Thin Python driver over the C++ host mirror (include/pbrt_host.h).

Names follow the reference's scene-description calls (src/core/api.rs): Material, Shape
"trianglemesh", AreaLightSource, LookAt, Camera, Film, Sampler, Integrator, WorldEnd -> render.
All numerics live in the C++/CUDA library; this file only marshals numpy arrays.
"""
import ctypes as C

import numpy as np

from . import _abi


class PbrtError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("pbrt status %d: %s" % (code, msg))
        self.code = code


def _fptr(a):
    return a.ctypes.data_as(C.POINTER(C.c_float)) if a is not None else None


def _f32(a, shape=None):
    if a is None:
        return None
    a = np.ascontiguousarray(a, dtype=np.float32)
    if shape is not None:
        a = a.reshape(shape)
    return a


class HostScene:
    """Mirrors the API state machine of src/core/api.rs for the in-scope directives."""

    def __init__(self, lib=None):
        self.L = lib if lib is not None else _abi.load()  # `lib`: tests may pass another build of the same C ABI
        self.h = self.L.pbrt_host_new()
        self._keep = []
        self.n_tris = 0
        # the same directives, recorded in call order, so that the scene can be written out as .pbrt text for a real rs_pbrt build
        # (rs_pbrt_b200/pbrt_export.py); (name, dict of arguments) tuples
        self.log = []

    def close(self):
        if self.h:
            self.L.pbrt_host_free(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _ck(self, rc):
        if rc < 0:
            raise PbrtError(rc, self.L.pbrt_host_last_error().decode())
        return rc

    def material(self, kind, params, textures=None, bump=None):
        """`textures`: {parameter group: texture index} (the group table in include/pbrt_gpu.h; e.g. matte {0: kd_tex, 1: sigma_tex})."""
        self.log.append(("material", dict(kind=int(kind), params=[float(x) for x in params], textures=dict(textures or {}), bump=bump)))
        p = np.zeros(24, np.float32)
        p[: len(params)] = np.asarray(params, np.float32)
        m = self._ck(self.L.pbrt_host_add_material(self.h, kind, _fptr(p)))
        for group, tex in (textures or {}).items():
            self._ck(self.L.pbrt_host_material_texture(self.h, m, int(group), int(tex)))
        if bump is not None:  # "texture bumpmap": a float texture
            self._ck(self.L.pbrt_host_material_bump(self.h, m, int(bump)))
        return m

    def material_mix(self, m1, m2, amount=(0.5, 0.5, 0.5)):
        """Material "mix" over two earlier materials (src/materials/mixmat.rs): m1's lobes scaled by amount, m2's by 1 - amount."""
        a = np.zeros(3, np.float32)
        a[:] = np.asarray(amount, np.float32)
        self.log.append(("material_mix", dict(m1=int(m1), m2=int(m2), amount=[float(x) for x in a])))
        return self._ck(self.L.pbrt_host_add_material_mix(self.h, int(m1), int(m2), _fptr(a)))

    def texture_image(self, rgb, trilinear=False, max_anisotropy=8.0, wrap=0, scale=1.0, gamma=False, uscale=1.0, vscale=1.0, udelta=0.0,
                      vdelta=0.0, float_valued=False):
        """Texture "spectrum" | "float" "imagemap": rgb = (height, width, 3) in [0,1], row 0 = top of the image as a decoder delivers it.
        `float_valued`: an ImageTexture<Float> (the luminance of the converted texels), for sigma / roughness / index parameters."""
        t = np.ascontiguousarray(rgb, np.float32)
        assert t.ndim == 3 and t.shape[2] == 3
        self.log.append(("texture_image", dict(rgb=t.copy(), trilinear=bool(trilinear), max_anisotropy=float(max_anisotropy), wrap=int(wrap), scale=float(scale), gamma=bool(gamma),
                                               uscale=float(uscale), vscale=float(vscale), udelta=float(udelta), vdelta=float(vdelta), float_valued=bool(float_valued))))
        return self._ck(self.L.pbrt_host_add_texture_image(self.h, _fptr(t), t.shape[1], t.shape[0], int(bool(float_valued)), int(bool(trilinear)), float(max_anisotropy),
                                                           int(wrap), float(scale), int(bool(gamma)), float(uscale), float(vscale), float(udelta),
                                                           float(vdelta)))

    def texture_mapping(self, texture, mapping, m):
        """"mapping" "spherical" / "cylindrical" (m: 4x4 world_to_texture) or "planar" (m: v1, v2) of an image texture."""
        kind = {"spherical": 1, "cylindrical": 2, "planar": 3}[mapping]
        a = np.ascontiguousarray(m, np.float32).reshape(-1)
        self.log.append(("texture_mapping", dict(texture=int(texture), mapping=mapping, m=a.copy())))
        assert a.size == (6 if kind == 3 else 16)
        self._ck(self.L.pbrt_host_texture_mapping(self.h, int(texture), kind, _fptr(a)))
        return texture

    def texture_constant(self, value, float_valued=False):
        """Texture "constant": a spectrum (3 values) or, with float_valued, one float."""
        v = np.zeros(3, np.float32)
        v[:] = np.asarray(value, np.float32)
        self.log.append(("texture_constant", dict(value=v.copy(), float_valued=bool(float_valued))))
        return self._ck(self.L.pbrt_host_add_texture_constant(self.h, _fptr(v), int(bool(float_valued))))

    def texture_scale(self, tex1, tex2):
        """Texture "scale": tex1 * tex2."""
        self.log.append(("texture_scale", dict(tex1=int(tex1), tex2=int(tex2))))
        return self._ck(self.L.pbrt_host_add_texture_scale(self.h, int(tex1), int(tex2)))

    def texture_mix(self, tex1, tex2, amount):
        """Texture "mix": tex1 * (1 - amount) + tex2 * amount, `amount` a float texture."""
        self.log.append(("texture_mix", dict(tex1=int(tex1), tex2=int(tex2), amount=int(amount))))
        return self._ck(self.L.pbrt_host_add_texture_mix(self.h, int(tex1), int(tex2), int(amount)))

    def trianglemesh(self, indices, P, N=None, S=None, UV=None, material=-1, emit=None, two_sided=False, reverse_orientation=False,
                     swaps_handedness=False):
        idx = np.ascontiguousarray(indices, dtype=np.uint32).reshape(-1)
        P = _f32(P, (-1, 3))
        N = _f32(N, (-1, 3))
        S = _f32(S, (-1, 3))
        UV = _f32(UV, (-1, 2))
        e = _f32(emit)
        self.n_tris += idx.size // 3
        self.log.append(("trianglemesh", dict(indices=idx.copy(), P=P.copy(), N=None if N is None else N.copy(), S=None if S is None else S.copy(), UV=None if UV is None else UV.copy(),
                                              material=int(material), emit=None if e is None else e.copy(), two_sided=bool(two_sided),
                                              reverse_orientation=bool(reverse_orientation), swaps_handedness=bool(swaps_handedness))))
        return self._ck(self.L.pbrt_host_add_trianglemesh(
            self.h, idx.size // 3, idx.ctypes.data_as(C.POINTER(C.c_uint32)), P.shape[0], _fptr(P), _fptr(N), _fptr(S), _fptr(UV),
            int(reverse_orientation), int(swaps_handedness), int(material), _fptr(e), int(two_sided)))

    def mesh_alpha(self, mesh, alpha=None, shadow_alpha=None):
        """Shape "texture alpha" / "texture shadowalpha": float textures (texture_image(float_valued=True), texture_constant(0, True), ...)."""
        self.log.append(("mesh_alpha", dict(mesh=int(mesh), alpha=alpha, shadow_alpha=shadow_alpha)))
        self._ck(self.L.pbrt_host_mesh_alpha(self.h, int(mesh), -1 if alpha is None else int(alpha), -1 if shadow_alpha is None else int(shadow_alpha)))
        return mesh

    def light_point(self, frm, I, scale=None):
        """LightSource "point" (api.rs make_light)."""
        f, i, sc = _f32(frm), _f32(I), _f32(scale)
        self.log.append(("light_point", dict(frm=f.copy(), I=i.copy(), scale=None if sc is None else sc.copy())))
        self._ck(self.L.pbrt_host_add_light_point(self.h, _fptr(f), _fptr(i), _fptr(sc)))

    def light_spot(self, frm, to, I, scale=None, coneangle=30.0, conedeltaangle=5.0):
        """LightSource "spot"."""
        f, t, i, sc = _f32(frm), _f32(to), _f32(I), _f32(scale)
        self.log.append(("light_spot", dict(frm=f.copy(), to=t.copy(), I=i.copy(), scale=None if sc is None else sc.copy(), coneangle=float(coneangle), conedeltaangle=float(conedeltaangle))))
        self._ck(self.L.pbrt_host_add_light_spot(self.h, _fptr(f), _fptr(t), _fptr(i), _fptr(sc), coneangle, conedeltaangle))

    def light_distant(self, frm, to, L, scale=None):
        """LightSource "distant" (direction = from - to)."""
        f, t, l, sc = _f32(frm), _f32(to), _f32(L), _f32(scale)
        self.log.append(("light_distant", dict(frm=f.copy(), to=t.copy(), L=l.copy(), scale=None if sc is None else sc.copy())))
        self._ck(self.L.pbrt_host_add_light_distant(self.h, _fptr(f), _fptr(t), _fptr(l), _fptr(sc)))

    def light_infinite(self, L, scale=None, texels=None, light_to_world=None):
        """LightSource "infinite": constant (texels=None) or an (h, w, 3) lat-long map; light_to_world = 3x3 rotation (CTM)."""
        l, sc = _f32(L), _f32(scale)
        self.log.append(("light_infinite", dict(L=l.copy(), scale=None if sc is None else sc.copy(), texels=None if texels is None else np.array(texels, np.float32),
                                                light_to_world=None if light_to_world is None else np.array(light_to_world, np.float32).reshape(3, 3))))
        w = h = 0
        t = None
        if texels is not None:
            t = _f32(texels)
            h, w = t.shape[0], t.shape[1]
            t = t.reshape(-1)
        m = mi = None
        if light_to_world is not None:
            m = _f32(light_to_world, (3, 3))
            mi = _f32(m.T.copy())  # a rotation: the reference carries the transpose as the inverse (transform.rs rotate)
            m = m.reshape(-1)
            mi = mi.reshape(-1)
        self._ck(self.L.pbrt_host_add_light_infinite(self.h, _fptr(l), _fptr(sc), _fptr(t), w, h, _fptr(m), _fptr(mi)))

    def look_at(self, eye, look, up):
        e, l, u = (_f32(v) for v in (eye, look, up))
        self.log.append(("look_at", dict(eye=e.copy(), look=l.copy(), up=u.copy())))
        self._ck(self.L.pbrt_host_look_at(self.h, _fptr(e), _fptr(l), _fptr(u)))

    def transform_times(self, start=0.0, end=1.0):
        """TransformTimes: the times of the start and end keyframes of every animated transform."""
        self.log.append(("transform_times", dict(start=float(start), end=float(end))))
        self._ck(self.L.pbrt_host_transform_times(self.h, start, end))

    def camera_motion(self, camera_to_world_end):
        """The camera's end keyframe (camera-to-world at the end time, 4x4); the start keyframe is look_at's.  None = static."""
        m = _f32(camera_to_world_end, (4, 4)) if camera_to_world_end is not None else None
        self.log.append(("camera_motion", dict(m=None if m is None else m.copy())))
        self._ck(self.L.pbrt_host_camera_motion(self.h, _fptr(m.reshape(-1)) if m is not None else None))

    def film(self, xres, yres, crop=None, filter="box", xwidth=0.5, ywidth=0.5, alpha=2.0, max_sample_luminance=float("inf")):
        c = _f32(crop)
        self.log.append(("film", dict(xres=int(xres), yres=int(yres), crop=None if c is None else c.copy(), filter=filter, xwidth=float(xwidth), ywidth=float(ywidth), alpha=float(alpha),
                                      max_sample_luminance=float(max_sample_luminance))))
        self._ck(self.L.pbrt_host_film(self.h, xres, yres, _fptr(c), filter.encode(), xwidth, ywidth, alpha, max_sample_luminance))

    def camera(self, fov=90.0, lensradius=0.0, focaldistance=1e6, shutteropen=0.0, shutterclose=1.0, screenwindow=None):
        sw = _f32(screenwindow)
        self.log.append(("camera", dict(fov=float(fov), lensradius=float(lensradius), focaldistance=float(focaldistance), shutteropen=float(shutteropen), shutterclose=float(shutterclose),
                                        screenwindow=None if sw is None else sw.copy())))
        self._ck(self.L.pbrt_host_camera_perspective(self.h, fov, lensradius, focaldistance, shutteropen, shutterclose, _fptr(sw)))

    def sampler(self, pixelsamples=16, name="sobol", samplepixelcenter=False):
        """Sampler "sobol" (pixelsamples rounded up to a power of two) or "halton"."""
        self.log.append(("sampler", dict(pixelsamples=int(pixelsamples), name=name, samplepixelcenter=bool(samplepixelcenter))))
        if name == "halton":
            self._ck(self.L.pbrt_host_sampler_halton(self.h, pixelsamples, int(samplepixelcenter)))
        elif name == "sobol":
            self._ck(self.L.pbrt_host_sampler_sobol(self.h, pixelsamples))
        else:
            raise ValueError("sampler outside the GPU path: %s" % name)

    def object_begin(self):
        """ObjectBegin: meshes added until object_end() belong to the returned object."""
        self.log.append(("object_begin", {}))
        return self._ck(self.L.pbrt_host_object_begin(self.h))

    def object_end(self):
        self.log.append(("object_end", {}))
        self._ck(self.L.pbrt_host_object_end(self.h))

    def object_instance(self, obj, instance_to_world=None):
        """ObjectInstance with the given 4x4 instance-to-world matrix (None = identity)."""
        self.log.append(("object_instance", dict(obj=int(obj), m=None if instance_to_world is None else np.array(instance_to_world, np.float32).reshape(4, 4))))
        m = _f32(instance_to_world, (4, 4)) if instance_to_world is not None else None
        self._ck(self.L.pbrt_host_object_instance(self.h, obj, _fptr(m.reshape(-1)) if m is not None else None))

    def instancing(self, mode):
        """"reference" (TransformedPrimitive::intersect as written, quirk Q7) or "fixed" (pbrt-v3)."""
        self.log.append(("instancing", dict(mode=mode)))
        self._ck(self.L.pbrt_host_instancing(self.h, {"reference": 0, "fixed": 1}[mode]))

    def integrator_direct(self, maxdepth=5, strategy="all", pixelbounds=None):
        """Integrator "directlighting"."""
        self.log.append(("integrator", dict(name="directlighting", maxdepth=int(maxdepth), strategy=strategy, pixelbounds=pixelbounds)))
        pb = np.ascontiguousarray(pixelbounds, np.int32) if pixelbounds is not None else None
        self._ck(self.L.pbrt_host_integrator_direct(self.h, maxdepth, {"all": 0, "one": 1}[strategy],
                                                    pb.ctypes.data_as(C.POINTER(C.c_int32)) if pb is not None else None))

    def integrator_whitted(self, maxdepth=5, pixelbounds=None):
        """Integrator "whitted"."""
        self.log.append(("integrator", dict(name="whitted", maxdepth=int(maxdepth), pixelbounds=pixelbounds)))
        pb = np.ascontiguousarray(pixelbounds, np.int32) if pixelbounds is not None else None
        self._ck(self.L.pbrt_host_integrator_whitted(self.h, maxdepth, pb.ctypes.data_as(C.POINTER(C.c_int32)) if pb is not None else None))

    def light_samples(self, n):
        """"nsamples" of the light sources declared after this call (DirectLightingIntegrator strategy "all")."""
        self.log.append(("light_samples", dict(n=int(n))))
        self._ck(self.L.pbrt_host_light_samples(self.h, int(n)))

    def integrator_ao(self, nsamples=64, cossample=True):
        """Integrator "ao"."""
        self.log.append(("integrator", dict(name="ao", nsamples=int(nsamples), cossample=bool(cossample))))
        self._ck(self.L.pbrt_host_integrator_ao(self.h, nsamples, int(cossample)))

    def integrator(self, maxdepth=5, rrthreshold=1.0, lightsamplestrategy="spatial", pixelbounds=None):
        self.log.append(("integrator", dict(name="path", maxdepth=int(maxdepth), rrthreshold=float(rrthreshold), lightsamplestrategy=lightsamplestrategy, pixelbounds=pixelbounds)))
        strat = {"uniform": 0, "power": 1, "spatial": 2}[lightsamplestrategy]
        pb = np.ascontiguousarray(pixelbounds, np.int32) if pixelbounds is not None else None
        self._ck(self.L.pbrt_host_integrator_path(self.h, maxdepth, rrthreshold, strat,
                                                  pb.ctypes.data_as(C.POINTER(C.c_int32)) if pb is not None else None))

    def world_end(self, maxnodeprims=4, n_threads=8):
        self.log.append(("world_end", dict(maxnodeprims=int(maxnodeprims))))
        self._ck(self.L.pbrt_host_world_end(self.h, maxnodeprims, n_threads))

    @property
    def desc(self):
        return self.L.pbrt_host_scene_desc(self.h)

    @property
    def params(self):
        return self.L.pbrt_host_render_params(self.h)

    @property
    def motion(self):
        """The PbrtMotionDesc of the built scene, or None when nothing in it is animated."""
        p = self.L.pbrt_host_motion_desc(self.h)
        return p if p else None

    def film_shape(self):
        cb = self.params.contents.cropped_pixel_bounds
        return (cb[3] - cb[1], cb[2] - cb[0])

    def render(self, device=0, rect=None):
        """Integrator::render: scene upload + GPU render + film merge.  Returns PbrtStats as a dict."""
        st = _abi.PbrtStats()
        r = np.ascontiguousarray(rect, np.int32) if rect is not None else None
        self._ck(self.L.pbrt_host_render(self.h, device, r.ctypes.data_as(C.POINTER(C.c_int32)) if r is not None else None, C.byref(st)))
        return st.as_dict()

    def film_rgbw(self):
        h, w = self.film_shape()
        p = self.L.pbrt_host_film_rgbw(self.h)
        return np.ctypeslib.as_array(p, shape=(h, w, 4)).copy()

    def film_clear(self):
        self._ck(self.L.pbrt_host_film_clear(self.h))

    def film_add(self, rgbw):
        a = _f32(rgbw)
        self._ck(self.L.pbrt_host_film_add_rgbw(self.h, _fptr(a)))

    def film_rgb(self):
        h, w = self.film_shape()
        out = np.zeros((h, w, 3), np.float32)
        self._ck(self.L.pbrt_host_film_rgb(self.h, _fptr(out)))
        return out

    def write_image(self, path):
        self._ck(self.L.pbrt_host_write_image(self.h, str(path).encode()))


class GpuScene:
    """A scene resident on one GPU: pbrt_gpu_scene_create / render / intersect (include/pbrt_gpu.h).  `motion`: a PbrtMotionDesc (or a
    pointer to one, e.g. HostScene.motion) for pbrt_gpu_scene_create_motion."""

    def __init__(self, desc, device=0, lib=None, motion=None):
        self.L = lib if lib is not None else _abi.load()  # `lib`: tests may pass another build of the same C ABI
        self.handle = C.c_void_p()
        if motion is not None:
            rc = self.L.pbrt_gpu_scene_create_motion(desc, motion if isinstance(motion, C._Pointer) else C.byref(motion), device, C.byref(self.handle))
        else:
            rc = self.L.pbrt_gpu_scene_create(desc, device, C.byref(self.handle))
        if rc != 0:
            raise PbrtError(rc, self.L.pbrt_gpu_last_error().decode())

    def upload_bytes(self):
        return int(self.L.pbrt_gpu_scene_bytes(self.handle))

    def close(self):
        if self.handle:
            self.L.pbrt_gpu_scene_destroy(self.handle)
            self.handle = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _ck(self, rc):
        if rc != 0:
            raise PbrtError(rc, self.L.pbrt_gpu_last_error().decode())

    @staticmethod
    def _rect(params, rect):
        r = np.ascontiguousarray(rect if rect is not None else list(params.contents.sample_bounds), np.int32)
        return r

    def render(self, params, rect=None, film=None):
        cb = params.contents.cropped_pixel_bounds
        if film is None:
            film = np.zeros((cb[3] - cb[1], cb[2] - cb[0], 4), np.float32)
        r = self._rect(params, rect)
        st = _abi.PbrtStats()
        self._ck(self.L.pbrt_gpu_render(self.handle, params, r.ctypes.data_as(C.POINTER(C.c_int32)), _fptr(film), C.byref(st)))
        return film, st.as_dict()

    def render_device(self, params, d_film_ptr, rect=None, stream=None):
        r = self._rect(params, rect)
        st = _abi.PbrtStats()
        self._ck(self.L.pbrt_gpu_render_device(self.handle, params, r.ctypes.data_as(C.POINTER(C.c_int32)), C.c_void_p(d_film_ptr),
                                               C.c_void_p(stream or 0), C.byref(st)))
        return st.as_dict()

    def render_tiles_device(self, params, d_film_ptr, part, n_parts, stream=None):
        """This rank's interleaved share of the frame's 16x16 tiles (Morton order, tile t -> part t mod n_parts) into a device film."""
        st = _abi.PbrtStats()
        self._ck(self.L.pbrt_gpu_render_tiles_device(self.handle, params, int(part), int(n_parts), C.c_void_p(d_film_ptr), C.c_void_p(stream or 0), C.byref(st)))
        return st.as_dict()

    def render_samples(self, params, rect):
        r = self._rect(params, rect)
        n = (r[2] - r[0]) * (r[3] - r[1])
        out = np.zeros((r[3] - r[1], r[2] - r[0], params.contents.spp, 3), np.float32)
        st = _abi.PbrtStats()
        if n > 0:
            self._ck(self.L.pbrt_gpu_render_samples(self.handle, params, r.ctypes.data_as(C.POINTER(C.c_int32)), _fptr(out), C.byref(st)))
        return out, st.as_dict()

    def intersect(self, o, d, t_max=None):
        o, d = _f32(o, (-1, 3)), _f32(d, (-1, 3))
        n = o.shape[0]
        tm = _f32(t_max) if t_max is not None else np.full(n, np.inf, np.float32)
        prim = np.zeros(n, np.int32)
        t = np.zeros(n, np.float32)
        b = np.zeros((n, 3), np.float32)
        st = _abi.PbrtStats()
        self._ck(self.L.pbrt_gpu_intersect(self.handle, n, _fptr(o), _fptr(d), _fptr(tm), prim.ctypes.data_as(C.POINTER(C.c_int32)),
                                           _fptr(t), _fptr(b), C.byref(st)))
        return prim, t, b, st.as_dict()

    def intersect_p(self, o, d, t_max=None):
        o, d = _f32(o, (-1, 3)), _f32(d, (-1, 3))
        n = o.shape[0]
        tm = _f32(t_max) if t_max is not None else np.full(n, np.inf, np.float32)
        occ = np.zeros(n, np.uint8)
        st = _abi.PbrtStats()
        self._ck(self.L.pbrt_gpu_intersect_p(self.handle, n, _fptr(o), _fptr(d), _fptr(tm), occ.ctypes.data_as(C.POINTER(C.c_uint8)),
                                             C.byref(st)))
        return occ, st.as_dict()


def pin_description(desc, lib=None):
    """pbrt_gpu_host_register on the big arrays of a scene description (nodes, tris, every mesh's p / n / s / uv), as a caller that
    re-creates the scene for every frame would do once; returns the handle `unpin_description` takes."""
    L = lib if lib is not None else _abi.load()
    d = desc.contents
    arrays = [(C.cast(d.nodes, C.c_void_p).value, 32 * d.n_nodes), (C.cast(d.tris, C.c_void_p).value, 24 * d.n_tris)]
    for i in range(d.n_meshes):
        m = d.meshes[i]
        for ptr, width in ((m.p, 12), (m.n, 12), (m.s, 12), (m.uv, 8)):
            a = C.cast(ptr, C.c_void_p).value
            if a:
                arrays.append((a, width * m.n_verts))
    done = []
    for a, n in arrays:
        if a and n >= (1 << 16) and L.pbrt_gpu_host_register(C.c_void_p(a), n) == 0:  # (small arrays are not worth a registration)
            done.append(a)
    return L, done


def unpin_description(handle):
    L, done = handle
    for a in done:
        L.pbrt_gpu_host_unregister(C.c_void_p(a))


def render_multi(gpu_scenes, params, film=None):
    """pbrt_gpu_render_multi: one frame on several devices from this process (one GpuScene per device), into a host film."""
    L = gpu_scenes[0].L
    cb = params.contents.cropped_pixel_bounds
    if film is None:
        film = np.zeros((cb[3] - cb[1], cb[2] - cb[0], 4), np.float32)
    handles = (C.c_void_p * len(gpu_scenes))(*[g.handle for g in gpu_scenes])
    st = _abi.PbrtStats()
    rc = L.pbrt_gpu_render_multi(handles, len(gpu_scenes), params, _fptr(film), C.byref(st))
    if rc != 0:
        raise PbrtError(rc, L.pbrt_gpu_last_error().decode())
    return film, st.as_dict()


def bvh_build(bounds, max_prims_in_node=4, n_threads=1):
    """BVHAccel::new on (n, 6) float32 bounds through the host mirror.  Returns (nodes structured array, ordered)."""
    L = _abi.load()
    b = _f32(bounds, (-1, 6))
    n = b.shape[0]
    nodes = (_abi.PbrtBvhNode * max(2 * n, 1))()
    ordered = np.zeros(max(n, 1), np.uint32)
    nn = C.c_uint32(0)
    rc = L.pbrt_host_bvh_build(_fptr(b), n, max_prims_in_node, n_threads, nodes, C.byref(nn), ordered.ctypes.data_as(C.POINTER(C.c_uint32)))
    if rc != 0:
        raise PbrtError(rc, L.pbrt_host_last_error().decode())
    arr = np.frombuffer(nodes, dtype=np.uint8)[: nn.value * 32].reshape(nn.value, 32).copy()
    return arr, ordered[:n].copy()
