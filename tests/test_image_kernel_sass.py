"""CPU test of the image kernels' machine code in the built library (sm_90a SASS, read with cuobjdump): the 64-bit
cell updates are done with native 32-bit shared-memory atomics, with no compare-and-swap loop left."""
import os
import re
import shutil
import subprocess

import pytest

from gpd_b200 import lib

CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"


def cuobjdump(flag):
    if not os.path.exists(CUOBJDUMP):
        pytest.skip("cuobjdump is not installed")
    return subprocess.run([CUOBJDUMP, flag, lib.SO_PATH], check=True, capture_output=True, text=True).stdout


def test_no_64bit_shared_atomic_loops_in_image_kernels():
    # "Function : <mangled name>" opens each kernel's SASS
    parts = re.split(r"^\s*Function\s*:\s*(\S+)\s*$", cuobjdump("-sass"), flags=re.M)
    fs = {n: body for n, body in zip(parts[1::2], parts[2::2]) if "k_images" in n}
    assert len(fs) >= 2 + 8  # k_images2<BATCH> and k_images<S, GL, BATCH>
    for n, body in fs.items():
        assert "ATOMS.CAST.SPIN.64" not in body, n

