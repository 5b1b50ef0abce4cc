"""The step kernel's shared-memory budget: how many envs (warps) one block holds for the bench scene.

Each env keeps its working set in a slice of dynamic shared memory (fe_layout_build, fe_engine.h) followed by the env's
FE_ENV_EXTRA_WORDS; a block holds as many slices as fit in 227 KB less 1 KB, at most FE_MAX_WPB (plat_prepare,
fe_host.cpp).  Sawyer + table_lack_0825 at its calibrated contact capacity must fit 16 per block: 132 x 16 = 2112 env slots
per launch on an H100, so 4096 envs run in two rounds instead of three.  The layout is the same function in the
lane-emulated build, so this is checked without a GPU."""
from furniture_b200 import mjcf
from parity_util import make_engine

SMEM_PER_BLOCK = 227 * 1024 - 1024  # what plat_prepare shares out among the warps of a block
MAX_WPB = 16  # FE_MAX_WPB
EXTRA_WORDS = 64  # FE_ENV_EXTRA_WORDS


def warps_per_block(bytes_per_env):
    return min(SMEM_PER_BLOCK // bytes_per_env, MAX_WPB)


def test_bench_scene_fits_16_envs_per_block():
    m = mjcf.load_scene("Sawyer", "table_lack_0825")
    eng = make_engine(m, 2, False)
    per_env = eng.L.fe_smem_bytes_per_env(eng.h)
    slice_words = per_env // 4 - EXTRA_WORDS
    print("Sawyer + table_lack_0825: slice %d words, %d bytes per env" % (slice_words, per_env))
    assert slice_words <= 3552
    assert 16 * per_env <= SMEM_PER_BLOCK
    assert warps_per_block(per_env) == 16


def test_larger_models_still_fit_a_block():
    """the models with the most dofs still get at least one warp per block"""
    for agent, furniture in [("Baxter", "table_lack_0825"), ("Sawyer", "bookcase_expedit_0385")]:
        m = mjcf.load_scene(agent, furniture)
        eng = make_engine(m, 1, False)
        assert warps_per_block(eng.L.fe_smem_bytes_per_env(eng.h)) >= 1
