"""TEST INFRASTRUCTURE: tests/pbrt_reader.py extended to the Camera directives other than "perspective" that
rs_pbrt_b200/pbrt_export.py writes ("orthographic", "environment"), with their shutter, lens and screen window.  The base reader
turns every Camera directive into HostScene.camera (a perspective camera); here the scene it builds is a HostScene whose camera()
makes the camera the file names."""
import re
from pathlib import Path

import pbrt_reader
from rs_pbrt_b200 import HostScene


def camera_directive(path):
    """-> (camera name, {parameter: value or [values]}) of the file's Camera directive."""
    text = "\n".join(l.split("#")[0] for l in Path(path).read_text().splitlines())
    m = re.search(r'^\s*Camera\s+"(\w+)"(.*)$', text, re.M)
    name, rest = m.group(1), m.group(2)
    ps = pbrt_reader._params(pbrt_reader.TOK.findall(rest))
    return name, {n: (v[1] if n == "screenwindow" else v[1][0]) for n, v in ps.items()}


def read(path, n_threads=4):
    name, c = camera_directive(path)
    shutter = dict(shutteropen=c.get("shutteropen", 0.0), shutterclose=c.get("shutterclose", 1.0))

    class CameraHost(HostScene):
        def camera(self, fov=90.0, lensradius=0.0, focaldistance=1e6, shutteropen=0.0, shutterclose=1.0, screenwindow=None):
            if name == "orthographic":
                self.camera_orthographic(lensradius=lensradius, focaldistance=focaldistance, screenwindow=screenwindow, **shutter)
            elif name == "environment":
                self.camera_environment(**shutter)
            else:
                super().camera(fov=fov, lensradius=lensradius, focaldistance=focaldistance, screenwindow=screenwindow, **shutter)

    saved = pbrt_reader.HostScene
    pbrt_reader.HostScene = CameraHost
    try:
        return pbrt_reader.read(path, n_threads=n_threads)
    finally:
        pbrt_reader.HostScene = saved
