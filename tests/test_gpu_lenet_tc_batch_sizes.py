"""The wgmma LeNet at batch sizes around the grid size (-m gpu): each CTA of conv2 walks a grid-stride sequence of
image tiles through a converter / two-consumer pipeline, so a batch smaller than the SM count, a single image and
batches that leave CTAs with unequal image counts must give the same per-image logits as a large batch."""
import numpy as np
import pytest

from gpd_b200 import lib, scenes

pytestmark = pytest.mark.gpu


def test_tensor_core_lenet_is_batch_size_independent():
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    rng = np.random.default_rng(7)
    n = 2 * sms + 3
    imgs = rng.integers(0, 256, (n, 60, 60, 15), dtype=np.uint8)
    w = scenes.random_lenet_weights(15, seed=15)
    out = {}
    for impl in (0, 1):
        ctx = lib.Context(lib.default_params(channels=15, lenet_impl=impl))
        ctx.set_weights(w)
        out[impl] = ctx.classify(imgs)[1]
        if impl == 0:
            for m in (1, 2, sms - 1, sms + 1):
                part = ctx.classify(imgs[:m])[1]
                assert np.array_equal(part, out[0][:m]), m
        ctx.close()
    assert np.all(np.isfinite(out[0]))
    assert np.abs(out[0] - out[1]).max() <= 1e-4 * np.abs(out[1]).max()
