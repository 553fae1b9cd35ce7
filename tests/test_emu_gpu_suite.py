"""The -m gpu parity tests, at their GPU sizes, through the kernel emulation (tests/emu: the CUDA sources compiled by g++, a block's
threads as fibers of one host thread).  On the GPU box these tests are the parity tests proper; here the same files run against
librs_pbrt_b200_emu.so (RS_PBRT_B200_LIB), so that a change to kernel logic, queues, class plans or the C ABI that would fail them
on hardware fails the CPU suite first.  What this cannot show is in tests/emu/include/cuda_runtime.h (memory model, scheduling, nvcc's
code generation, performance).  Test infrastructure: nothing under rs_pbrt_b200/ loads the emulation library by itself."""
import os
import shutil
import subprocess
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
pytestmark = pytest.mark.skipif(shutil.which("g++") is None, reason="needs g++")

FILES = ["test_gpu_closed_forms.py", "test_gpu_parity_cornell.py", "test_gpu_parity_halton.py", "test_gpu_parity_lights.py", "test_gpu_parity_materials.py", "test_gpu_parity_siblings.py"]


@pytest.mark.parametrize("name", FILES)
def test_gpu_marked_file_passes_through_the_emulation(name):
    sys.path.insert(0, str(ROOT / "tests" / "emu"))
    import build_emu

    lib = build_emu.build()
    env = dict(os.environ, RS_PBRT_B200_LIB=str(lib))
    env.pop("PYTEST_XDIST_WORKER", None)
    r = subprocess.run([sys.executable, "-m", "pytest", str(ROOT / "tests" / name), "-q", "-x", "-m", "gpu", "-p", "no:xdist", "-p", "no:cacheprovider"],
                       cwd=ROOT, env=env, capture_output=True, text=True, timeout=1500)
    tail = "\n".join((r.stdout + r.stderr).splitlines()[-25:])
    assert r.returncode == 0, tail
    assert " passed" in tail and "failed" not in tail, tail


@pytest.mark.parametrize("knobs", ["PB_BATCH_LOG2=10 PB_STREAMS=2", "PB_BATCH_LOG2=10 PB_RAY_SORT=2", "PB_SHADE_SPEC=0 PB_BATCH_LOG2=11 PB_POLL_LAG=1"])
def test_scene_family_hunt_with_several_batches_per_frame(knobs):
    """The randomised scene families at four times the frame size under a 1024-sample batch limit: every frame is several batches (two in flight with
    PB_STREAMS=2), the batch borders fall inside pixels' sample runs and inside tiles.  The knobs are read once per process, hence the child process;
    the other two rows keep the experiment paths (two-level ray order, general k_shade only, late-polled loops) honest."""
    sys.path.insert(0, str(ROOT / "tests" / "emu"))
    import build_emu

    build_emu.build()
    env = dict(os.environ, RS_PBRT_FUZZ_GROW="4", RS_PBRT_FUZZ_FAMILIES="48", **dict(kv.split("=") for kv in knobs.split()))
    env.pop("PYTEST_XDIST_WORKER", None)
    r = subprocess.run([sys.executable, "-m", "pytest", str(ROOT / "tests" / "test_emu_kernels.py"), "-q", "-x", "-p", "no:xdist", "-p", "no:cacheprovider", "-k", "randomised_scene_families"],
                       cwd=ROOT, env=env, capture_output=True, text=True, timeout=1500)
    tail = "\n".join((r.stdout + r.stderr).splitlines()[-25:])
    assert r.returncode == 0 and "48 passed" in tail, tail
