"""TEST INFRASTRUCTURE: tests/pbrt_reader.py extended to the Camera "realistic" that rs_pbrt_b200/pbrt_export.py writes: its lens
file (read as read_float_file reads it), aperture, focus distance, weighting and shutter, and the Film's "diagonal".  The existing
readers are unchanged; the scene it builds is a HostScene whose camera() makes the realistic camera."""
import re
from pathlib import Path

import pbrt_reader
import pbrt_reader_cameras
from rs_pbrt_b200 import HostScene


def film_diagonal(path):
    """The Film directive's "float diagonal" in mm (35, film.rs:250, when absent)."""
    text = "\n".join(l.split("#")[0] for l in Path(path).read_text().splitlines())
    m = re.search(r'^\s*Film\s+"\w+"(.*)$', text, re.M)
    ps = pbrt_reader._params(pbrt_reader.TOK.findall(m.group(1)))
    return ps["diagonal"][1][0] if "diagonal" in ps else 35.0


def read_float_file(path):
    """read_float_file (src/core/floatfile.rs): every number of the file, `#` starting a comment."""
    return [float(t) for l in Path(path).read_text().splitlines() for t in l.split("#")[0].split()]


def read(path, n_threads=4):
    name, c = pbrt_reader_cameras.camera_directive(path)
    if name != "realistic":
        return pbrt_reader_cameras.read(path, n_threads=n_threads)
    sw = c.get("simpleweighting", "true")
    simple = (sw.strip('"') == "true") if isinstance(sw, str) else bool(sw)

    class RealisticHost(HostScene):
        def camera(self, fov=90.0, lensradius=0.0, focaldistance=1e6, shutteropen=0.0, shutterclose=1.0, screenwindow=None):
            self.film_diagonal(film_diagonal(path))
            self.camera_realistic(read_float_file(Path(path).parent / c["lensfile"].strip('"')), aperturediameter=c.get("aperturediameter", 1.0),
                                  focusdistance=c.get("focusdistance", 10.0), simpleweighting=simple, shutteropen=c.get("shutteropen", 0.0),
                                  shutterclose=c.get("shutterclose", 1.0))

    saved = pbrt_reader.HostScene
    pbrt_reader.HostScene = RealisticHost
    try:
        return pbrt_reader.read(path, n_threads=n_threads)
    finally:
        pbrt_reader.HostScene = saved
