"""k_sort finishes every slot of the shade queue that has no surface to shade -- the path ray missed, or the path already ended and only its
pending next-event estimate is left -- so k_shade visits surface hits only: its slot count (PbrtStats.shade_slots) equals the vertices it
shades, while the samples stay the oracle's.  Through the kernel emulation (tests/emu), like tests/test_emu_kernels.py."""
import shutil

import numpy as np
import pytest

from rs_pbrt_b200 import scenes
from test_emu_kernels import check, emu  # noqa: F401  (emu: the module-scoped fixture)

pytestmark = pytest.mark.skipif(shutil.which("g++") is None, reason="needs g++")


def _instances_under_a_sky(mode):
    import test_oracle_instancing as T

    return T.scene(mode, [np.eye(4, dtype=np.float32), T.translate(2, 0, 0)], wall=True, sky=np.array([0.25, 0.5, 1.0], np.float32), res=(10, 8), spp=2)


@pytest.mark.parametrize("make", [
    lambda: scenes.cornell_box(xres=12, yres=12, spp=2),                                   # area light only
    lambda: scenes.sky_scene(xres=10, yres=10, spp=2, env="two", strategy="spatial"),    # escaped paths and MIS rays pick up the environment
    lambda: scenes.cornell_box(xres=10, yres=10, spp=2, materials="mixed", lights="delta", strategy="power"),  # specular classes, delta lights
    lambda: _instances_under_a_sky("reference"),                                          # moved-instance hits filed under class 1 (quirk Q7)
], ids=["cornell", "sky", "mixed-delta", "instances-reference"])
def test_shade_kernel_visits_surface_hits_only(emu, oracle, make):  # noqa: F811
    st = check(emu, oracle, make(), count_work=True)
    assert st["shade_slots"] > 0
    assert st["shade_slots"] == st["shaded_vertices"]
