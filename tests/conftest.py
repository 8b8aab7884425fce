import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


@pytest.fixture(scope="session")
def golden_dir():
    return os.path.join(ROOT, "tests", "golden")


@pytest.fixture(scope="session")
def weights15():
    import numpy as np
    from oracle import oracle
    z = np.load(os.path.join(ROOT, "gpd_b200", "weights", "lenet_15ch.npz"))
    return [z[n] for n in oracle.WeightPack.NAMES]


def load_weights(ch):
    import numpy as np
    from oracle import oracle
    path = os.path.join(ROOT, "gpd_b200", "weights", f"lenet_{ch}ch.npz")
    if not os.path.exists(path):
        # the reference ships no 1-channel LeNet: random-init weights of its architecture (seeded) classify the
        # 1-channel images in the parity tests — oracle and kernels get the same arrays
        from gpd_b200 import scenes
        return scenes.random_lenet_weights(ch, seed=ch), 0
    z = np.load(path)
    return [z[n] for n in oracle.WeightPack.NAMES], int(z["relu_after_conv"])
