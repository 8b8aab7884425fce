"""The sequential host restatement of include/gpd_b200_train.h rules 1, 2 and 5 (tests/train_chains.cpp) on the CPU: on
its own float32 forward it stays within the float64 error bounds of train_reference; its pooling choices are the float64
first maximum wherever the float64 margin exceeds the chains' error; and departures a kernel rewrite could make (another
summation order, a chunked image chain, the last maximum on ties) each change bits, while the first three stay within
the bounds, which is why test_gpu_train_chains.py compares bits rather than bounds."""
import numpy as np
import pytest

import train_chains as tc
import train_reference as tr

F = np.float32
STAGE_INPUTS = ("pool1", "pool2", "ip1", "logits", "choice1", "choice2", "dlogits", "dip1", "dpool2", "dpool1")


def bits(a):
    return np.ascontiguousarray(a, F).view(np.uint32)


def own_step(images, labels, w, relu):
    """the restatement's step on its own float32 forward, with ip1 and the logits computed in float64 from its pool2 and
    rounded: the per-image arrays of gpdb_train_debug and the eight gradients"""
    C, n = images.shape[-1], len(labels)
    _, _, _, _, W1, B1, W2, B2 = tr.arrays64(w, C)
    d = {}
    d["choice1"], d["pool1"] = tc.pool1(images, w, relu)
    d["choice2"], d["pool2"] = tc.pool2(d["pool1"], w, relu)
    d["ip1"] = np.maximum(d["pool2"].astype(np.float64) @ W1 + B1, 0).astype(F)
    d["logits"] = (d["ip1"].astype(np.float64) @ W2 + B2).astype(F)
    d["loss"], d["dlogits"] = tr.host_loss(d["logits"], labels, n)
    d["dip1"] = tc.dip1(d["ip1"], d["dlogits"], w)
    d["dpool2"] = tc.dpool2(d["dip1"], w)
    d["dconv2"] = tc.dconv2(d["dpool2"], d["pool2"], d["choice2"], relu)
    d["dpool1"] = tc.dpool1(d["dconv2"], w)
    d["grad"] = tc.grads(images, d, relu)
    return d


def within(got, ref, bound):
    return bool((np.abs(np.asarray(got, np.float64) - ref) <= bound).all())


@pytest.mark.parametrize("n", [3, 17])
@pytest.mark.parametrize("relu", [0, 1])
@pytest.mark.parametrize("C", [1, 3, 12, 15])
def test_restatement_within_the_float64_bounds(C, relu, n):
    w = tr.random_net(C, seed=40 + C + relu)
    images = tr.random_images(n, C, seed=n + C, ties=(n + relu) % 2 == 1)
    labels = np.arange(n) % 2
    d = own_step(images, labels, w, relu)
    dev = {k: d[k] for k in STAGE_INPUTS}
    st = tr.backward64(images, labels, w, relu, dev)
    b = tr.bounds(images, labels, w, relu, st)
    for k in ("dip1", "dpool2", "dpool1"):
        assert within(d[k], st[k], b[k]), k
    ref, bnd = tr.step_grad_bounds(images, labels, w, relu, dev, slice_size=8)
    for i in range(8):
        assert within(d["grad"][i], ref[i], bnd[i]), i
        assert within(d["grad"][i], st["grad"][i], b["grad"][i]), i
        assert np.abs(d["grad"][i]).max() > 0, i


def _windows(v):
    """[n, o, 2P, 2P] -> [n, o, P, P, 4] in row-major window order"""
    n, o, H, W = v.shape
    return v.reshape(n, o, H // 2, 2, W // 2, 2).transpose(0, 1, 2, 4, 3, 5).reshape(n, o, H // 2, W // 2, 4)


def _decided(v, err):
    """where the float64 window values v are far enough apart for any float32 chains within err of them: the largest
    value exceeds every other by more than twice the window's largest error"""
    s = np.sort(v, -1)
    return s[..., 3] - s[..., 2] > 2 * err.max(-1)


@pytest.mark.parametrize("C", [1, 3, 12, 15])
def test_pooling_choices_are_the_float64_first_maximum(C):
    relu = C % 2
    w = tr.random_net(C, seed=60 + C)
    images = tr.random_images(4, C, seed=C, ties=True)
    w1, b1, w2, b2 = tr.arrays64(w, C)[:4]
    ch1, p1 = tc.pool1(images, w, relu)
    ch2, _ = tc.pool2(p1, w, relu)
    x = tr.chw(images)
    for ch, v, err in (
            (ch1, tr.conv(x, w1, b1), tr.gamma(25 * C + 1) * tr.conv(x, np.abs(w1), np.abs(b1))),
            (tr.unflat(ch2), tr.conv(p1.astype(np.float64), w2, b2),
             tr.gamma(501) * tr.conv(np.abs(p1.astype(np.float64)), np.abs(w2), np.abs(b2)))):
        v, err = _windows(v), _windows(err)
        ok = _decided(v, err)
        assert ok.mean() > 0.5, ok.mean()  # most windows are decided; the flat patches tie
        assert np.array_equal(ch[ok], v.argmax(-1)[ok])


def test_flat_images_choose_the_first_position():
    """every window of both pools ties on a flat image: the first position wins (the last-maximum variant takes 3)"""
    for C in (1, 15):
        w = tr.random_net(C, seed=C)
        images = np.full((2, 60, 60, C), 90, np.uint8)
        for relu in (0, 1):
            ch1, p1 = tc.pool1(images, w, relu)
            ch2, _ = tc.pool2(p1, w, relu)
            assert (ch1 == 0).all() and (ch2 == 0).all()
            assert (tc.pool1(images, w, relu, variant=1)[0] == 3).all()
            assert (tc.pool2(p1, w, relu, variant=1)[0] == 3).all()


def synthetic_step(n, C, seed):
    """per-image arrays of a step of n images with the shapes and signs of gpdb_train_debug's, drawn at random: the image
    chains of the gradients read them as given, so they need not come from one forward pass"""
    rng = np.random.default_rng(seed)
    r = lambda *s: rng.standard_normal(s).astype(F)  # noqa: E731
    d = {"pool1": np.maximum(r(n, 20, 28, 28), 0), "pool2": np.maximum(r(n, 7200), 0), "ip1": np.maximum(r(n, 500), 0),
         "logits": r(n, 2), "choice1": rng.integers(0, 4, (n, 20, 28, 28)).astype(np.uint8),
         "choice2": rng.integers(0, 4, (n, 7200)).astype(np.uint8), "dlogits": r(n, 2) / F(n), "dip1": r(n, 500) / F(n),
         "dpool2": r(n, 7200) / F(n), "dpool1": r(n, 20, 28, 28) / F(n)}
    return tr.random_images(n, C, seed=seed), rng.integers(0, 2, n), d


def test_departures_change_bits_the_bounds_let_through():
    C, relu = 1, 1
    w = tr.random_net(C, seed=70)
    # d pool1 chained over (kh, kw, o) instead of (o, kh, kw)
    images = tr.random_images(3, C, seed=71)
    labels = np.array([0, 1, 1])
    d = own_step(images, labels, w, relu)
    st = tr.backward64(images, labels, w, relu, {k: d[k] for k in STAGE_INPUTS})
    b = tr.bounds(images, labels, w, relu, st)
    other = tc.dpool1(d["dconv2"], w, variant=1)
    assert (bits(other) != bits(d["dpool1"])).any()
    assert within(other, st["dpool1"], b["dpool1"])

    # a step of 300 images: the conv gradients' image chain restarted at image 256 (two totals added), and dW1 chained
    # over the images in reverse
    n = 300
    images, labels, d = synthetic_step(n, C, seed=72)
    ref, bnd = tr.step_grad_bounds(images, labels, w, relu, d)
    g = tc.grads(images, d, relu)
    for i in range(8):
        assert within(g[i], ref[i], bnd[i]), i
    g1 = tc.conv1_grads(images, d["dpool1"], d["pool1"], d["choice1"], relu, restart=256)
    g2 = tc.conv2_grads(d["pool1"], d["dpool2"], d["pool2"], d["choice2"], relu, restart=256)
    for i, a in zip(range(4), (*g1, *g2)):
        assert (bits(a) != bits(g[i])).any(), i
        assert within(a, ref[i], bnd[i]), i
    assert np.array_equal(tc.conv1_grads(images, d["dpool1"], d["pool1"], d["choice1"], relu, restart=n)[0], g[0])
    rev = tc.ip_grads(d["pool2"], d["dip1"], d["ip1"], d["dlogits"], reverse=True)[0]
    assert (bits(rev) != bits(g[4])).any()
    assert within(rev, ref[4], bnd[4])

    # the last maximum instead of the first on ties: images with flat patches
    images = tr.random_images(2, C, seed=73, ties=True)
    ch1, p1 = tc.pool1(images, w, relu)
    assert (tc.pool1(images, w, relu, variant=1)[0] != ch1).any()
    assert (tc.pool2(p1, w, relu, variant=1)[0] != tc.pool2(p1, w, relu)[0]).any()
