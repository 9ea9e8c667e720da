import os
import sys

import pytest

# the C oracle uses OpenMP over matmul rows; on a 128-core GPU box the fork/join cost of 128 threads dwarfs the
# tiny test models, so cap it (results do not depend on the thread count)
os.environ.setdefault("OMP_NUM_THREADS", "8")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (sm_90a); run with -m gpu")


@pytest.fixture(scope="session")
def tmp_models(tmp_path_factory):
    """Directory with seeded synthetic slice files, created on demand (key -> path)."""
    from distributedllm_b200 import ggjt

    root = tmp_path_factory.mktemp("models")
    cache = {}

    def get(shape: str, wtype: int = ggjt.T_Q4_0, layer_from: int = 0, layer_to: int = 1, seed: int = 0) -> str:
        key = (shape, wtype, layer_from, layer_to, seed)
        if key not in cache:
            p = str(root / ("%s_%s_%d_%d_s%d.bin" % (shape, ggjt.TYPE_NAME[wtype], layer_from, layer_to, seed)))
            ggjt.write_synth_slice(p, ggjt.SHAPES[shape], layer_from, layer_to, wtype, seed)
            cache[key] = p
        return cache[key]

    return get
