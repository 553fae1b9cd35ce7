"""Write a HostScene out as .pbrt text (plus .ply meshes and .png / .hdr images) that a real rs_pbrt build can render.

This is the bridge from "parity unpinned" to a pinned oracle (SURVEY.md section 8c/8d): rs_pbrt cannot be built in this image (no
Rust toolchain, no crates), so the reference itself never runs here -- but every synthetic scene of `rs_pbrt_b200/scenes.py` can leave
the building as the input rs_pbrt reads, and `tools/compare_with_rs_pbrt.py` renders it with `rs_pbrt --integrator path` wherever a
toolchain exists and compares the float film.  Grammar: /root/reference/examples/rs_pbrt.pest; CLI: src/bin/rs_pbrt.rs:41-68.

    from rs_pbrt_b200 import scenes, pbrt_export
    h = scenes.cornell_box(xres=400, yres=400, spp=64)
    pbrt_export.write(h, "out/cornell.pbrt")

The directives come from `HostScene.log` (every HostScene call is recorded in order).  Meshes are in world space already (the host
mirror takes world-space vertices, like api.rs does after applying the CTM), so the file has no transforms except the instances'.
What cannot be carried exactly is said in the returned notes: rs_pbrt reads textures through the `image` crate as 8-bit RGB
(imagemap.rs:44-57), so an exported float texture is quantised (generate scenes with `quantize_textures=True` to have both sides
agree), and environment maps go out as Radiance .hdr (RGBE).
"""
import struct
import zlib
from pathlib import Path

import numpy as np

MATERIALS = {  # kind -> (pbrt name, [(parameter, n values, params[] offset)], texture groups in pbrt_gpu.h order, remap offset)
    0: ("matte", [("Kd", 3, 0), ("sigma", 1, 3)], ["Kd", "sigma"], None),
    1: ("plastic", [("Kd", 3, 0), ("Ks", 3, 3), ("roughness", 1, 6)], ["Kd", "Ks", "roughness"], 7),
    2: ("metal", [("eta", 3, 0), ("k", 3, 3), ("uroughness", 1, 6), ("vroughness", 1, 7)], ["eta", "k", "uroughness", "vroughness"], 8),
    3: ("mirror", [("Kr", 3, 0)], ["Kr"], None),
    4: ("glass", [("Kr", 3, 0), ("Kt", 3, 3), ("index", 1, 6), ("uroughness", 1, 7), ("vroughness", 1, 8)], ["Kr", "Kt", "index", "uroughness", "vroughness"], 9),
    5: ("uber", [("Kd", 3, 0), ("Ks", 3, 3), ("Kr", 3, 6), ("Kt", 3, 9), ("opacity", 3, 12), ("uroughness", 1, 15), ("vroughness", 1, 16), ("index", 1, 17)],
        ["Kd", "Ks", "Kr", "Kt", "opacity", "uroughness", "vroughness", "index"], 18),
    6: ("substrate", [("Kd", 3, 0), ("Ks", 3, 3), ("uroughness", 1, 6), ("vroughness", 1, 7)], ["Kd", "Ks", "uroughness", "vroughness"], 8),
    7: ("translucent", [("Kd", 3, 0), ("Ks", 3, 3), ("reflect", 3, 6), ("transmit", 3, 9), ("roughness", 1, 12)], ["Kd", "Ks", "reflect", "transmit", "roughness"], 13),
}
WRAP = {0: "repeat", 1: "black", 2: "clamp"}


def _nums(a):
    return " ".join(repr(float(x)) for x in np.asarray(a, np.float64).reshape(-1))


def _ints(a):
    return " ".join(str(int(x)) for x in np.asarray(a).reshape(-1))


def write_png(path, rgb8):
    """Minimal 8-bit RGB PNG (zlib only)."""
    h, w, _ = rgb8.shape
    raw = b"".join(b"\x00" + rgb8[y].tobytes() for y in range(h))

    def chunk(tag, data):
        c = struct.pack(">I", len(data)) + tag + data
        return c + struct.pack(">I", zlib.crc32(tag + data) & 0xFFFFFFFF)

    Path(path).write_bytes(b"\x89PNG\r\n\x1a\n" + chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, 8, 2, 0, 0, 0)) + chunk(b"IDAT", zlib.compress(raw, 6)) + chunk(b"IEND", b""))


def write_hdr(path, rgb):
    """Radiance RGBE, uncompressed scanlines, top row first."""
    h, w, _ = rgb.shape
    m = np.max(rgb, axis=2)
    e = np.where(m > 1e-32, np.floor(np.log2(np.maximum(m, 1e-38))) + 1, 0.0)
    scale = np.where(m > 1e-32, 256.0 / np.exp2(e), 0.0)
    out = np.zeros((h, w, 4), np.uint8)
    out[..., :3] = np.clip(rgb * scale[..., None], 0, 255).astype(np.uint8)
    out[..., 3] = np.where(m > 1e-32, e + 128, 0).astype(np.uint8)
    Path(path).write_bytes(b"#?RADIANCE\nFORMAT=32-bit_rle_rgbe\n\n" + ("-Y %d +X %d\n" % (h, w)).encode() + out.tobytes())


def write_ply(path, idx, P, N=None, UV=None):
    """Binary little-endian PLY as src/shapes/plymesh.rs reads it (x y z [nx ny nz] [u v], vertex_indices lists)."""
    n = P.shape[0]
    props = ["property float x", "property float y", "property float z"]
    cols = [P.astype("<f4")]
    if N is not None:
        props += ["property float nx", "property float ny", "property float nz"]
        cols.append(N.astype("<f4"))
    if UV is not None:
        props += ["property float u", "property float v"]
        cols.append(UV.astype("<f4"))
    header = "ply\nformat binary_little_endian 1.0\nelement vertex %d\n%s\nelement face %d\nproperty list uchar int vertex_indices\nend_header\n" % (
        n, "\n".join(props), idx.size // 3)
    faces = np.zeros(idx.size // 3, dtype=[("n", "u1"), ("v", "<i4", 3)])
    faces["n"] = 3
    faces["v"] = idx.reshape(-1, 3)
    Path(path).write_bytes(header.encode() + np.concatenate(cols, axis=1).tobytes() + faces.tobytes())


def write(h, path, ply_threshold=2000):
    """Write `h` (a HostScene after world_end) to `path`; returns a list of notes about what could not be carried exactly."""
    path = Path(path)
    path.parent.mkdir(parents=True, exist_ok=True)
    stem = path.stem
    notes = []
    pre, world = [], []
    materials, textures, tex_names = [], [], []
    mesh_attrs = {}  # mesh index -> (alpha texture, shadow alpha texture)
    n_mesh = 0
    for name, a in h.log:  # alpha masks are declared after their mesh: collect them first
        if name == "trianglemesh":
            n_mesh += 1
        elif name == "mesh_alpha":
            mesh_attrs[a["mesh"]] = (a["alpha"], a["shadow_alpha"])

    def tex_decl(i):
        t = textures[i]
        nm = tex_names[i]
        kind = "float" if t.get("float_valued") else "spectrum"
        if t["type"] == "image":
            img = np.clip(t["rgb"], 0.0, 1.0)
            q = np.round(img * 255.0).astype(np.uint8)
            if np.abs(q.astype(np.float32) / 255.0 - img).max() > 1e-7:
                notes.append("texture %s: texels quantised to 8 bits (rs_pbrt reads images through to_rgb8, imagemap.rs:44-57)" % nm)
            write_png(path.parent / ("%s_%s.png" % (stem, nm)), q)
            s = 'Texture "%s" "%s" "imagemap" "string filename" ["%s_%s.png"] "bool trilinear" ["%s"] "float maxanisotropy" [%r] "string wrap" ["%s"] "float scale" [%r] "bool gamma" ["%s"]' % (
                nm, kind, stem, nm, "true" if t["trilinear"] else "false", t["max_anisotropy"], WRAP[t["wrap"]], t["scale"], "true" if t["gamma"] else "false")
            mp = t.get("mapping")
            if mp is None:
                s += ' "float uscale" [%r] "float vscale" [%r] "float udelta" [%r] "float vdelta" [%r]' % (t["uscale"], t["vscale"], t["udelta"], t["vdelta"])
            elif mp[0] == "planar":
                s += ' "string mapping" ["planar"] "vector v1" [%s] "vector v2" [%s] "float udelta" [%r] "float vdelta" [%r]' % (_nums(mp[1][:3]), _nums(mp[1][3:6]), t["udelta"], t["vdelta"])
            else:  # spherical / cylindrical: world_to_texture is the CTM at the Texture directive
                s = "AttributeBegin\n  Transform [%s]\n  %s \"string mapping\" [\"%s\"]\nAttributeEnd" % (_nums(np.asarray(mp[1]).reshape(4, 4).T), s, mp[0])
            return s
        if t["type"] == "constant":
            v = t["value"]
            return 'Texture "%s" "%s" "constant" %s' % (nm, kind, ('"float value" [%r]' % float(v[0])) if t["float_valued"] else ('"rgb value" [%s]' % _nums(v)))
        if t["type"] == "scale":
            return 'Texture "%s" "%s" "scale" "texture tex1" "%s" "texture tex2" "%s"' % (nm, kind, tex_names[t["tex1"]], tex_names[t["tex2"]])
        return 'Texture "%s" "%s" "mix" "texture tex1" "%s" "texture tex2" "%s" "texture amount" "%s"' % (nm, kind, tex_names[t["tex1"]], tex_names[t["tex2"]], tex_names[t["amount"]])

    def material_decl(m, named=None):
        """`Material "<kind>" ...`, or with `named` the same material as `MakeNamedMaterial "<named>" "string type" ["<kind>"] ...`."""
        if m.get("mix"):  # api.rs:678-705: the children are named materials of the current graphics state (mix_decls below declares them first)
            head = 'MakeNamedMaterial "%s" "string type" ["mix"]' % named if named else 'Material "mix"'
            return '%s "string namedmaterial1" ["mat%d"] "string namedmaterial2" ["mat%d"] "rgb amount" [%s]' % (head, m["m1"], m["m2"], _nums(m["amount"]))
        name, plist, groups, remap = MATERIALS[m["kind"]]
        p = list(m["params"]) + [0.0] * 24
        parts = ['MakeNamedMaterial "%s" "string type" ["%s"]' % (named, name) if named else 'Material "%s"' % name]
        bound = {groups[g]: t for g, t in m["textures"].items()}
        for pn, nv, off in plist:
            if pn in bound:
                parts.append('"texture %s" "%s"' % (pn, tex_names[bound[pn]]))
            elif nv == 3:
                parts.append('"rgb %s" [%s]' % (pn, _nums(p[off:off + 3])))
            else:
                parts.append('"float %s" [%r]' % (pn, float(p[off])))
        if remap is not None:
            parts.append('"bool remaproughness" ["%s"]' % ("true" if p[remap] != 0.0 else "false"))
        if m["bump"] is not None:
            parts.append('"texture bumpmap" "%s"' % tex_names[m["bump"]])
        return " ".join(parts)

    def mix_decls(i, declared):
        """MakeNamedMaterial lines for everything the mix material `i` names, children before parents ("mat<index>")."""
        lines = []
        for c in (materials[i]["m1"], materials[i]["m2"]):
            if c in declared:
                continue
            declared.add(c)
            if materials[c].get("mix"):
                lines += mix_decls(c, declared)
            lines.append(material_decl(materials[c], named="mat%d" % c))
        return lines

    light_samples = 1
    mesh_i = 0
    in_object = False
    objects = 0
    film = sampler = integrator = camera = look = camera_end = times = None
    for name, a in h.log:
        if name == "material":
            materials.append(a)
        elif name == "material_mix":
            materials.append(dict(a, mix=True))
        elif name.startswith("texture_"):
            if name == "texture_mapping":
                textures[a["texture"]]["mapping"] = (a["mapping"], a["m"])
                continue
            t = dict(a)
            t["type"] = name[len("texture_"):]
            if t["type"] in ("scale", "mix"):
                t["float_valued"] = textures[t["tex1"]].get("float_valued", False)
            textures.append(t)
            tex_names.append("tex%d" % (len(textures) - 1))
        elif name == "light_samples":
            light_samples = a["n"]
        elif name == "trianglemesh":
            out = ["AttributeBegin"]
            if a["material"] >= 0 and materials[a["material"]].get("mix"):  # (named materials live in the graphics state: they end with this attribute block)
                out += ["  " + l for l in mix_decls(a["material"], set())]
            out.append("  " + (material_decl(materials[a["material"]]) if a["material"] >= 0 else 'Material "none"'))
            if a["emit"] is not None:
                out.append('  AreaLightSource "diffuse" "rgb L" [%s] "bool twosided" ["%s"] "integer samples" [%d]' % (_nums(a["emit"]), "true" if a["two_sided"] else "false", light_samples))
            if a["reverse_orientation"]:
                out.append("  ReverseOrientation")
            if a["swaps_handedness"]:
                notes.append("mesh %d: transform_swaps_handedness set by hand cannot be expressed without a mirroring transform" % mesh_i)
            extra = ""
            al = mesh_attrs.get(mesh_i)
            if al:
                if al[0] is not None:
                    extra += ' "texture alpha" "%s"' % tex_names[al[0]]
                if al[1] is not None:
                    extra += ' "texture shadowalpha" "%s"' % tex_names[al[1]]
            if a["S"] is not None:
                notes.append("mesh %d: per-vertex tangents (S) are only read from inline trianglemesh shapes" % mesh_i)
            if a["P"].shape[0] > ply_threshold and a["S"] is None:
                fn = "%s_mesh%d.ply" % (stem, mesh_i)
                write_ply(path.parent / fn, a["indices"], a["P"], a["N"], a["UV"])
                out.append('  Shape "plymesh" "string filename" ["%s"]%s' % (fn, extra))
            else:
                s = '  Shape "trianglemesh" "integer indices" [%s] "point P" [%s]' % (_ints(a["indices"]), _nums(a["P"]))
                if a["N"] is not None:
                    s += ' "normal N" [%s]' % _nums(a["N"])
                if a["S"] is not None:
                    s += ' "vector S" [%s]' % _nums(a["S"])
                if a["UV"] is not None:
                    s += ' "float uv" [%s]' % _nums(a["UV"])
                out.append(s + extra)
            out.append("AttributeEnd")
            world.append("\n".join(("  " + l if in_object else l) for l in out))
            mesh_i += 1
        elif name == "object_begin":
            world.append('ObjectBegin "obj%d"' % objects)
            in_object = True
        elif name == "object_end":
            world.append("ObjectEnd")
            in_object = False
            objects += 1
        elif name == "object_instance":
            if a["m"] is None:
                world.append('ObjectInstance "obj%d"' % a["obj"])
            else:
                world.append('AttributeBegin\n  Transform [%s]\n  ObjectInstance "obj%d"\nAttributeEnd' % (_nums(a["m"].T), a["obj"]))
        elif name == "light_point":
            world.append('LightSource "point" "point from" [%s] "rgb I" [%s]%s' % (_nums(a["frm"]), _nums(a["I"]), "" if a["scale"] is None else ' "rgb scale" [%s]' % _nums(a["scale"])))
        elif name == "light_spot":
            world.append('LightSource "spot" "point from" [%s] "point to" [%s] "rgb I" [%s] "float coneangle" [%r] "float conedeltaangle" [%r]%s' % (
                _nums(a["frm"]), _nums(a["to"]), _nums(a["I"]), a["coneangle"], a["conedeltaangle"], "" if a["scale"] is None else ' "rgb scale" [%s]' % _nums(a["scale"])))
        elif name == "light_distant":
            world.append('LightSource "distant" "point from" [%s] "point to" [%s] "rgb L" [%s]%s' % (_nums(a["frm"]), _nums(a["to"]), _nums(a["L"]), "" if a["scale"] is None else ' "rgb scale" [%s]' % _nums(a["scale"])))
        elif name == "light_infinite":
            s = 'LightSource "infinite" "rgb L" [%s] "integer samples" [%d]' % (_nums(a["L"]), light_samples)
            if a["scale"] is not None:
                s += ' "rgb scale" [%s]' % _nums(a["scale"])
            if a["texels"] is not None:
                fn = "%s_env%d.hdr" % (stem, len(world))
                write_hdr(path.parent / fn, np.asarray(a["texels"], np.float32))
                notes.append("environment map %s: written as Radiance RGBE (8-bit mantissas)" % fn)
                s += ' "string mapname" ["%s"]' % fn
            if a["light_to_world"] is not None:
                m4 = np.eye(4, dtype=np.float32)
                m4[:3, :3] = a["light_to_world"]
                s = "AttributeBegin\n  Transform [%s]\n  %s\nAttributeEnd" % (_nums(m4.T), s)
            world.append(s)
        elif name == "look_at":
            look = "LookAt %s  %s  %s" % (_nums(a["eye"]), _nums(a["look"]), _nums(a["up"]))
        elif name == "transform_times":
            times = a
        elif name == "camera_motion":
            camera_end = a["m"]
        elif name == "film":
            film = a
        elif name == "camera":
            camera = a
        elif name == "sampler":
            sampler = a
        elif name == "integrator":
            integrator = a
        elif name == "instancing" and a["mode"] != "reference":
            notes.append('instancing "fixed" (pbrt-v3 behaviour) is a library switch; rs_pbrt itself renders the "reference" behaviour (quirk Q7)')
    if times:
        pre.append("TransformTimes %r %r" % (times["start"], times["end"]))
    if camera_end is not None:  # the CTM at the Camera directive is world_to_camera: the end keyframe goes in as its inverse
        notes.append("camera end keyframe: written as the f32 inverse of camera_to_world, which rs_pbrt inverts again")
        w2c_end = np.linalg.inv(np.asarray(camera_end, np.float64)).astype(np.float32)
        pre += ["ActiveTransform StartTime"] + ([look] if look else []) + ["ActiveTransform EndTime", "Transform [%s]" % _nums(w2c_end.T), "ActiveTransform All"]
    elif look:
        pre.append(look)
    c = camera or {}
    s = 'Camera "perspective" "float fov" [%r]' % c.get("fov", 90.0)
    if (c.get("shutteropen", 0.0), c.get("shutterclose", 1.0)) != (0.0, 1.0):
        s += ' "float shutteropen" [%r] "float shutterclose" [%r]' % (c["shutteropen"], c["shutterclose"])
    if c.get("lensradius", 0.0) > 0.0:
        s += ' "float lensradius" [%r] "float focaldistance" [%r]' % (c["lensradius"], c["focaldistance"])
    if c.get("screenwindow") is not None:
        s += ' "float screenwindow" [%s]' % _nums(c["screenwindow"])
    pre.append(s)
    sp = sampler or dict(name="sobol", pixelsamples=16, samplepixelcenter=False)
    pre.append('Sampler "%s" "integer pixelsamples" [%d]%s' % (sp["name"], sp["pixelsamples"], ' "bool samplepixelcenter" ["true"]' if sp.get("samplepixelcenter") else ""))
    it = integrator or dict(name="path", maxdepth=5, rrthreshold=1.0, lightsamplestrategy="spatial", pixelbounds=None)
    if it["name"] == "path":
        s = 'Integrator "path" "integer maxdepth" [%d] "float rrthreshold" [%r] "string lightsamplestrategy" ["%s"]' % (it["maxdepth"], it["rrthreshold"], it["lightsamplestrategy"])
    elif it["name"] == "ao":
        s = 'Integrator "ao" "integer nsamples" [%d] "bool cossample" ["%s"]' % (it["nsamples"], "true" if it["cossample"] else "false")
    elif it["name"] == "directlighting":
        s = 'Integrator "directlighting" "integer maxdepth" [%d] "string strategy" ["%s"]' % (it["maxdepth"], it["strategy"])
    else:
        s = 'Integrator "whitted" "integer maxdepth" [%d]' % it["maxdepth"]
    if it.get("pixelbounds") is not None:
        s += ' "integer pixelbounds" [%s]' % _ints(it["pixelbounds"])
    pre.append(s)
    f = film or dict(xres=1280, yres=720, crop=None, filter="box", xwidth=0.5, ywidth=0.5, alpha=2.0, max_sample_luminance=float("inf"))
    pre.append('PixelFilter "%s" "float xwidth" [%r] "float ywidth" [%r]%s' % (f["filter"], f["xwidth"], f["ywidth"], ' "float alpha" [%r]' % f["alpha"] if f["filter"] == "gaussian" else ""))
    s = 'Film "image" "integer xresolution" [%d] "integer yresolution" [%d] "string filename" ["%s.png"]' % (f["xres"], f["yres"], stem)
    if f.get("crop") is not None:
        s += ' "float cropwindow" [%s]' % _nums(f["crop"])
    if np.isfinite(f.get("max_sample_luminance", float("inf"))):
        s += ' "float maxsampleluminance" [%r]' % f["max_sample_luminance"]
    pre.append(s)
    text = ["# written by rs_pbrt_b200/pbrt_export.py: the synthetic stand-in scene of the same name, for `rs_pbrt --path %s`" % path.name] + pre + ["WorldBegin"]
    text += [tex_decl(i) for i in range(len(textures))]
    text += world + ["WorldEnd", ""]
    path.write_text("\n".join(text))
    return sorted(set(notes))
