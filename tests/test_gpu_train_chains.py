"""Every chain of a training step pinned bit for bit (-m gpu, include/gpd_b200_train.h rules 1, 2, 4 and 5).

One gpdb_debug_train_step per case returns the device's forward state, per-image stages and gradients. The sequential
host restatement (tests/train_chains.cpp) recomputes each stage on the device's own input to it, with the header's
chains in the header's order, so the comparison is exact:
- every image: the loss within 8 ulp and the d logits within 8 ulp of p / n of the header's helpers compiled for the host
  (the device's expf and log1pf are not libm's), and the eight gradients bit for bit;
- the pooling choices, pool1, pool2, d ip1, d pool2 and d pool1 bit for bit on the images around the edges of k_gemm's
  16-image stages and 64-row tiles and of the 256-image chunks, plus four seeded ones;
- the gradients within the float64 error bounds of train_reference.backward64, and once against torch float64 autograd,
  which do not depend on the restatement.
Then a train_step on the same images is the SGD update of the debug call's gradient, bit for bit, with the debug call's
mean loss. The sizes cross every stage, tile and chunk edge; every shipped channel count and both ReLU settings run.
A last test sets the logits through ip2's biases at the gaps where expf underflows.
"""
import functools

import numpy as np
import pytest

import train_chains as tc
import train_reference as tr
from conftest import load_weights
from gpd_b200 import lib, scenes

pytestmark = pytest.mark.gpu

F = np.float32
LR, MU = 1e-3, 0.9
EDGES = (0, 1, 15, 16, 17, 63, 64, 65, 255, 256, 257)
STAGES = ("choice1", "pool1", "choice2", "pool2", "dip1", "dpool2", "dpool1")
INPUTS = ("pool1", "pool2", "ip1", "logits", "choice1", "choice2", "dlogits", "dip1", "dpool2", "dpool1")
DEAD = (2, 9, 17)  # conv1 filters of the "dead3" net whose biases sit near -1e4
TORCH_CASE = "shipped3-257"

# (net, n, images): random images alternate ties=True / False down the table
TABLE = ([("shipped15", n) for n in (1, 16, 17, 64, 65, 256, 257, 513)] +
         [(f"shipped{C}", n) for C in (3, 12) for n in (17, 257)] +
         [(f"random1_relu{r}", n) for r in (0, 1) for n in (15, 300)] +
         [("random15_relu1", 65), ("dead3", 65)])
CASES = [(net, n, "ties" if k % 2 == 0 else "plain") for k, (net, n) in enumerate(TABLE)] + [("shipped15", 257, "grasp")]
IDS = [f"{net}-{n}" + ("-grasp" if im == "grasp" else "") for net, n, im in CASES]


@functools.lru_cache(None)
def net(name):
    """(C, the eight .bin arrays as float32, relu_after_conv)"""
    if name.startswith("shipped"):
        C = int(name[7:])
        w, relu = load_weights(C)
    elif name.startswith("random"):
        C, relu = int(name[6:name.index("_")]), int(name[-1])
        w = tr.random_net(C, seed=7 + relu if C == 1 else 3)
    else:  # a random 3-channel net with ReLU whose DEAD filters pool to exactly 0 on every image
        C, relu = 3, 1
        w = tr.random_net(C, seed=5)
        w[1] = w[1].copy()
        w[1][list(DEAD)] = F(-1e4) + np.arange(len(DEAD), dtype=F)
    return C, tuple(np.ascontiguousarray(np.asarray(a, F).ravel()) for a in w), relu


CAMS4 = np.array([[0.0, 0.0, 0.0], [0.6, 0.0, 0.0], [-0.6, 0.0, 0.0], [0.0, 0.6, 0.0]])


def grasp_batch(C, n):
    """The INTEGRATION recipe (as test_gpu_train.labelled_batch): candidates of one camera's view of each synthetic table
    scene, labelled against four-camera ground truths; the first positives, at most ceil(n / 2) of them, and then the
    first negatives, n images in all."""
    import torch
    p = lib.default_params(channels=C)
    seeds = tuple(range(3, 13))
    views = [scenes.synthetic_table_scene(s, n_points=20000) for s in seeds]
    gts = [scenes.synthetic_table_scene(s, n_points=20000, cameras=CAMS4, mark_all_cameras=True) for s in seeds]
    a, b = lib.Context(p), lib.Context(p)
    a.set_clouds(views)
    b.set_clouds(gts)
    sidx = [np.random.default_rng(s).choice(20000, 1000, replace=False).astype(np.int32) for s in range(len(seeds))]
    soff, idx = lib.pack_samples(sidx)
    rec, _, hoff = a.hand_search_batch_tensors(soff, torch.from_numpy(idx).cuda())
    images = a.images_batch_tensors(hoff, rec)
    labels = (b.reevaluate_batch_tensors(hoff, rec) == 1).to(torch.int32)
    pos = (labels == 1).nonzero().flatten()[: (n + 1) // 2]
    neg = (labels == 0).nonzero().flatten()[: n - len(pos)]
    assert len(pos) > 0 and len(pos) + len(neg) == n, (len(pos), len(neg))
    sel = torch.cat([pos, neg])
    return images[sel].cpu().numpy(), labels[sel].cpu().numpy().astype(np.int32)


def batch(kind, C, n, seed):
    if kind == "grasp":
        return grasp_batch(C, n)
    images = tr.random_images(n, C, seed=seed, ties=kind == "ties")
    return images, np.random.default_rng(seed).integers(0, 2, n).astype(np.int32)


def trainer(C, w, relu):
    ctx = lib.Context(lib.default_params(channels=C, relu_after_conv=relu))
    ctx.train_begin(lib.train_params(optimizer="sgd", lr=LR, momentum=MU), init=list(w))
    return ctx


def bits(a):
    return np.ascontiguousarray(a, F).view(np.uint32)


def assert_bits(got, want, what):
    g, r = bits(got), bits(want)
    bad = np.flatnonzero(g.ravel() != r.ravel())
    assert len(bad) == 0, (what, f"{len(bad)} of {g.size} differ", [(int(e), float(np.ravel(got)[e]), float(np.ravel(want)[e]))
                                                                 for e in bad[:4]])


def ulp(a, b):
    """bit-pattern distance of float32 arrays; 2^32 where the signs differ"""
    a, b = bits(a).astype(np.int64), bits(b).astype(np.int64)
    return np.where((a >> 31) == (b >> 31), np.abs(a - b), 2 ** 32)


def assert_ulp(got, want, what, limit=8):
    d = ulp(got, want)
    e = int(np.argmax(d))
    assert d.max() <= limit, (what, int(d.max()), float(np.ravel(got)[e]), float(np.ravel(want)[e]))


def assert_dlogits(got, z, labels, n, what="dlogits"):
    """rule 4 against the header's helper on the same logits: each d logit within 8 ulp of the larger of |dz_k| and
    p_k / n. When k is the labelled, larger logit, dz_k = (p_k - 1) / n cancels the leading bits of p_k, so a 1-ulp
    difference between the device's expf and libm's can be many ulp of dz_k itself (63 at a logit gap of 4.1)."""
    _, want = tr.host_loss(z, labels, n)
    p = np.stack(tr.probs_f32(np.asarray(z, F)), 1)
    tol = 8 * np.spacing(np.maximum(np.abs(want), p / F(n)).astype(F)).astype(np.float64)
    err = np.abs(got.astype(np.float64) - want)
    e = np.unravel_index(int(np.argmax(err / tol)), err.shape)
    assert (err <= tol).all(), (what, float(err[e] / tol[e] * 8), float(got[e]), float(want[e]), z[e[0]].tolist())


def subset(n, seed):
    """the images whose per-image stages are checked: every stage, tile and chunk edge below n, the last image and four
    seeded ones"""
    return np.unique([i for i in EDGES if i < n] + [n - 1] + list(np.random.default_rng(seed).integers(0, n, 4)))


def assert_grads_within_bounds(images, labels, w, relu, d):
    """the device's eight gradients within tr.bounds of tr.backward64 on the device's own stage inputs"""
    ref, bnd = tr.step_grad_bounds(images, labels, w, relu, {k: d[k] for k in INPUTS})
    for i in range(8):
        err = np.abs(d["grad"][i].astype(np.float64) - ref[i])
        assert (err <= bnd[i]).all(), (i, float((err / bnd[i]).max()))


@pytest.mark.parametrize("name,n,kind", CASES, ids=IDS)
def test_step_equals_the_host_chains(name, n, kind):
    C, w, relu = net(name)
    seed = 1000 + CASES.index((name, n, kind))
    images, labels = batch(kind, C, n, seed)
    t = trainer(C, w, relu)
    d = t.debug_train_step(images, labels)

    # rules 3 and 4 against the header's helpers on the device's logits
    assert_ulp(d["loss"], tr.host_loss(d["logits"], labels, n)[0], "loss")
    assert_dlogits(d["dlogits"], d["logits"], labels, n)

    # rule 5: the eight gradients of the whole step
    g = tc.grads(images, d, relu)
    for i in range(8):
        assert_bits(d["grad"][i], g[i], f"grad[{i}]")

    # rules 1, 2 and 5: the per-image stages, each on the device's input to it
    idx = subset(n, seed)
    st = tc.stages(images[idx], {k: d[k][idx] for k in INPUTS}, w, relu)
    for k in STAGES:
        if k.startswith("choice"):
            assert np.array_equal(d[k][idx], st[k]), k
        else:
            assert_bits(d[k][idx], st[k], k)

    assert_grads_within_bounds(images, labels, w, relu, d)
    if f"{name}-{n}" == TORCH_CASE and kind != "grasp":
        _, _, gt = tr.torch_grads64(images, labels, w, relu)
        for i in range(8):
            rel = np.linalg.norm(d["grad"][i] - gt[i]) / max(np.linalg.norm(gt[i]), 1e-30)
            assert rel <= 1e-4, (i, rel)
    if name == "dead3":
        assert (d["pool1"][:, list(DEAD)] == 0).all()
        nw = 3 * 25
        for o in DEAD:
            assert not d["grad"][0][o * nw:(o + 1) * nw].any() and d["grad"][1][o] == 0, o

    # the debug call updated nothing: a step on the same images is the SGD update of its gradient, with its mean loss
    got_loss = t.train_step(images, labels)
    assert F(got_loss).view(np.uint32) == tr.mean_loss_f32(d["loss"]).view(np.uint32)
    got = t.train_weights()
    for i in range(8):
        want, _ = tr.sgd_f32(w[i], d["grad"][i], np.zeros_like(w[i]), LR, MU, 0.0, True)
        assert_bits(got[i], want, f"sgd weights[{i}]")
    if n == 513:  # the device twin of a multi-chunk step: the same loss bits and weights
        import torch
        u = trainer(C, w, relu)
        lt = u.train_step_tensors(torch.from_numpy(images).cuda(), torch.from_numpy(labels).cuda())
        assert lt.cpu().numpy().view(np.uint32) == F(got_loss).view(np.uint32)
        for x, y in zip(u.train_weights(), got):
            assert_bits(x, y, "train_step_tensors weights")


GAPS = (0.0, 1e-30, 1.0, 88.0, 103.9, 104.0, 200.0)


@pytest.mark.parametrize("gap", GAPS)
def test_loss_and_dlogits_at_the_underflow_edges(gap):
    """ip2's weights 0 and its biases the logits: the device's loss and d logits within 8 ulp of the header's helpers at
    gaps where expf goes subnormal (88 .. 103.9) and then 0 (104, 200), for both labels and both orders of the logits;
    where the host's expf is 0, the d logits are exactly (p - y) / n with p = 1 for the larger logit and 0 for the other"""
    C, relu = 1, 0
    w = [np.asarray(a, F).ravel() for a in tr.random_net(C, seed=9)]
    w[6] = np.zeros(1000, F)
    images = tr.random_images(2, C, seed=4)
    labels = np.array([0, 1], np.int32)
    ctx = lib.Context(lib.default_params(channels=C, relu_after_conv=relu))
    for z in ((0.0, gap), (gap, 0.0)):
        w[7] = np.array(z, F)
        ctx.train_begin(lib.train_params(), init=w)
        d = ctx.debug_train_step(images, labels)
        assert np.array_equal(bits(d["logits"]), bits(np.tile(w[7], (2, 1)))), z
        assert_ulp(d["loss"], tr.host_loss(d["logits"], labels, 2)[0], ("loss", z))
        assert_dlogits(d["dlogits"], d["logits"], labels, 2, ("dlogits", z))
        if tr._vec("expf", [-abs(F(z[1]) - F(z[0]))])[0] == 0:
            p = np.array([0, 1] if z[1] >= z[0] else [1, 0], F)
            want = np.stack([(p - np.eye(2, dtype=F)[y]) / F(2) for y in labels])
            assert_bits(d["dlogits"], want, ("exact dlogits", z))
