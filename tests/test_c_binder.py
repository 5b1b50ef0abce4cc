"""A binder without Python: examples/step_from_c.c is compiled against include/furniture_b200.h and libfurniture_b200.so, creates its handle
from a compiled scene file (fe_create_from_file) and steps it with host buffers.  Without a GPU the program must end with the library's
error message and exit code 2 (no crash, no CPU fallback); on an H100 it steps."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIBDIR = os.path.join(ROOT, "furniture_b200")
SCENE = os.path.join(LIBDIR, "compiled", "Sawyer_table_lack_0825.feb")


@pytest.fixture(scope="module")
def binder(tmp_path_factory):
    if not os.path.exists(os.path.join(LIBDIR, "libfurniture_b200.so")):
        pytest.skip("CUDA library not built")
    exe = str(tmp_path_factory.mktemp("binder") / "step_from_c")
    subprocess.check_call(["gcc", "-O2", "-Wall", "-Werror", "-I" + os.path.join(ROOT, "include"), os.path.join(ROOT, "examples", "step_from_c.c"), "-o", exe,
                           "-L" + LIBDIR, "-lfurniture_b200", "-Wl,-rpath," + LIBDIR])
    return exe


def test_c_program_builds_against_the_header_and_fails_loudly_without_a_gpu(binder):
    from parity_util import have_gpu

    if have_gpu():
        pytest.skip("a GPU is present: covered by the gpu test")
    r = subprocess.run([binder, SCENE, "4", "1"], capture_output=True, text=True, timeout=120)
    assert r.returncode == 2 and "fe_create_from_file" in r.stderr and len(r.stderr.strip()) > 25, (r.returncode, r.stderr)
    r = subprocess.run([binder, os.path.join(ROOT, "README.md"), "4", "1"], capture_output=True, text=True, timeout=120)
    assert r.returncode == 2 and "scene file" in r.stderr  # not a scene file: said so before any device work


@pytest.mark.gpu
def test_c_program_steps_on_the_gpu(binder):
    r = subprocess.run([binder, SCENE, "64", "3"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    f = r.stdout.split()
    kv = dict(zip(f[0::2], f[1::2]))
    assert kv["envs"] == "64" and kv["obs_dim"] == "64" and kv["action_dim"] == "9" and kv["episode_length"] == "3" and kv["done"] == "0"
    assert abs(float(kv["mean_reward"]) + 1e-3 * 2) < 1e-4  # two action entries of magnitude 1: the control penalty of config/furniture.py:291
