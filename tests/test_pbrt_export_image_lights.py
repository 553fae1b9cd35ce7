"""The .pbrt export of goniometric and projection lights: LightSource "goniometric" / "projection" inside an attribute block with the
CTM, and the map as a Radiance .hdr whose first row is row 0 of the map (the reference's new_hdr does not flip rows)."""
import re

import numpy as np
import pytest

from rs_pbrt_b200 import pbrt_export, scenes


def read_hdr(path):
    data = path.read_bytes()
    head, _, rest = data.partition(b"\n\n")
    line, _, pix = rest.partition(b"\n")
    h, w = (int(v) for v in re.match(rb"-Y (\d+) \+X (\d+)", line).groups())
    px = np.frombuffer(pix, np.uint8).reshape(h, w, 4).astype(np.float64)
    return np.where(px[..., 3:] > 0, px[..., :3] * np.exp2(px[..., 3:] - 136.0), 0.0)


@pytest.mark.parametrize("kind", ["goniometric", "projection"])
def test_image_light_is_exported_with_its_ctm_and_map(tmp_path, kind):
    h = scenes.cornell_box(xres=8, yres=8, spp=1, lights=kind)
    pbrt_export.write(h, tmp_path / "scene.pbrt")
    text = (tmp_path / "scene.pbrt").read_text()
    m = re.search(r'AttributeBegin\s+Transform \[([^\]]*)\]\s+LightSource "%s" "rgb I" \[([^\]]*)\](.*?)\n' % kind, text)
    assert m, text[-2000:]
    entry = next(a for n, a in h.log if n == "light_" + kind)
    assert np.allclose(np.array(m.group(1).split(), np.float64).reshape(4, 4).T, entry["light_to_world"], rtol=1e-6)
    assert np.allclose(np.array(m.group(2).split(), np.float64), entry["I"])
    if kind == "projection":
        assert '"float fov" [%r]' % entry["fov"] in m.group(3)
    fn = re.search(r'"string mapname" \["([^"]+)"\]', m.group(3)).group(1)
    img = read_hdr(tmp_path / fn)
    assert img.shape == entry["texels"].shape
    t = entry["texels"].astype(np.float64)
    assert np.all(np.abs(img - t) <= t.max(-1, keepdims=True) / 128 + 1e-6)  # RGBE: 8-bit mantissas on the brightest channel's exponent
    assert np.array_equal(np.argmax(img.sum(-1)[:, 0]), np.argmax(t.sum(-1)[:, 0]))  # no row flip
