"""LeNet training on the device (-m gpu, include/gpd_b200_train.h): the training forward is gpdb_classify's with
lenet_impl = 1 bit for bit; every backward stage stays within its derived bound against the float64 restatement on the
device's own inputs; the whole gradient agrees with torch float64 autograd; the optimiser updates equal the numpy float32
restatement bit for bit; steps are deterministic and the twins agree; errors leave the state as it was; and a balanced
batch of candidate images made by the INTEGRATION recipe is overfitted."""
import numpy as np
import pytest

import train_reference as tr
from conftest import load_weights
from gpd_b200 import lib, scenes

pytestmark = pytest.mark.gpu

ERR_INVALID, ERR_STATE = -1, -3
F = np.float32


def nets():
    out = [(f"shipped{C}", C, *load_weights(C)) for C in (15, 3, 12)]
    out += [(f"random1_relu{r}", 1, tr.random_net(1, seed=7 + r), r) for r in (0, 1)]
    out += [("random15_relu0", 15, tr.random_net(15, seed=3), 0)]
    return out


NETS = nets()


def trainer(C, w, relu, **tp):
    ctx = lib.Context(lib.default_params(channels=C, relu_after_conv=relu))
    ctx.train_begin(lib.train_params(**tp), init=w)
    return ctx


def bits(a):
    return np.ascontiguousarray(a, F).view(np.uint32)


@pytest.mark.parametrize("name,C,w,relu", NETS, ids=[n[0] for n in NETS])
def test_forward_logits_equal_classify_simt(name, C, w, relu):
    cls = lib.Context(lib.default_params(channels=C, relu_after_conv=relu, lenet_impl=1))
    cls.set_weights(w)
    t = trainer(C, w, relu)
    sizes = (1, 63, 64, 65, tr.CHUNK - 1, tr.CHUNK) if name == "shipped15" else (1, 65)
    for n in sizes:
        images = tr.random_images(n, C, seed=n)
        labels = np.arange(n) % 2
        d = t.debug_train_step(images, labels)
        _, logits = cls.classify(images)
        assert np.array_equal(bits(d["logits"]), bits(logits)), n
    # a step of CHUNK + 1 images runs in two chunks: its loss is the mean over both of the classifier's logits
    n = tr.CHUNK + 1
    images, labels = tr.random_images(n, C, seed=n), np.arange(n) % 2
    _, logits = cls.classify(images)
    t0 = trainer(C, w, relu, lr=0.0, momentum=0.0)
    loss = t0.train_step(images, labels)
    ref = np.mean(np.logaddexp(logits[:, 0].astype(np.float64), logits[:, 1]) - logits[np.arange(n), labels])
    assert abs(loss - ref) <= 1e-5 * max(1.0, abs(ref))


@pytest.mark.parametrize("name,C,w,relu", NETS[:1] + NETS[3:], ids=[n[0] for n in NETS[:1] + NETS[3:]])
def test_backward_stages_within_bounds_and_gradient_against_torch(name, C, w, relu):
    n = 8
    images = tr.random_images(n, C, seed=11, ties=True)
    labels = np.array([0, 1] * 4)
    t = trainer(C, w, relu)
    d = t.debug_train_step(images, labels)
    st = tr.backward64(images, labels, w, relu, d)
    b = tr.bounds(images, labels, w, relu, st)
    for k in ("dlogits", "dip1", "dpool2", "dpool1"):
        err = np.abs(d[k].astype(np.float64) - st[k])
        assert (err <= b[k]).all(), (k, float((err / b[k]).max()))
    for i in range(8):
        err = np.abs(d["grad"][i].astype(np.float64) - st["grad"][i])
        assert (err <= b["grad"][i]).all(), (i, float((err / b["grad"][i]).max()))
    # the per-image losses against float64 on the device's logits (expf / log1pf within a few ulp)
    z = d["logits"].astype(np.float64)
    ref = np.logaddexp(z[:, 0], z[:, 1]) - z[np.arange(n), labels]
    assert np.allclose(d["loss"], ref, rtol=1e-6, atol=1e-6)
    # the whole gradient against torch float64 autograd from the same weights and images
    _, _, g = tr.torch_grads64(images, labels, w, relu)
    for i in range(8):
        rel = np.linalg.norm(d["grad"][i] - g[i]) / max(np.linalg.norm(g[i]), 1e-30)
        assert rel <= 1e-4, (i, rel)


@pytest.mark.parametrize("opt", [dict(optimizer="sgd", lr=1e-3, momentum=m, weight_decay=wd)
                                 for m in (0.0, 0.9) for wd in (0.0, 0.01)] +
                         [dict(optimizer="adam", lr=1e-3, weight_decay=wd) for wd in (0.0, 0.01)],
                         ids=["sgd_m0", "sgd_m0_wd", "sgd_m9", "sgd_m9_wd", "adam", "adam_wd"])
def test_optimiser_updates_equal_the_restatement(opt):
    C, relu = 3, 1
    w = [np.asarray(a, F).ravel() for a in tr.random_net(C, seed=21)]
    t = trainer(C, w, relu, **opt)
    p = [a.copy() for a in w]
    m = [np.zeros_like(a) for a in w]
    v = [np.zeros_like(a) for a in w]
    for step in range(1, 4):
        images, labels = tr.random_images(16, C, seed=100 + step), np.arange(16) % 2
        g = t.debug_train_step(images, labels)["grad"]
        t.train_step(images, labels)
        for i in range(8):
            if opt["optimizer"] == "sgd":
                p[i], m[i] = tr.sgd_f32(p[i], g[i], m[i], opt["lr"], opt["momentum"], opt["weight_decay"], step == 1)
            else:
                p[i], m[i], v[i] = tr.adam_f32(p[i], g[i], m[i], v[i], opt["lr"], 0.9, 0.999, 1e-8, opt["weight_decay"], step)
        got = t.train_weights()
        for i in range(8):
            assert np.array_equal(bits(got[i]), bits(p[i])), (step, i)


def test_determinism_and_twins():
    import torch
    C, relu = 15, 0
    w = load_weights(C)[0]
    rng = np.random.default_rng(0)
    images = tr.random_images(96, C, seed=1)
    labels = rng.integers(0, 2, 96).astype(np.int32)
    a, b = trainer(C, w, relu, optimizer="adam", lr=1e-4), trainer(C, w, relu, optimizer="adam", lr=1e-4)
    di, dl = torch.from_numpy(images).cuda(), torch.from_numpy(labels).cuda()
    for s in range(50):
        idx = np.random.default_rng(s).permutation(96)[:32]
        la = a.train_step(images[idx], labels[idx])
        lb = b.train_step_tensors(di[torch.from_numpy(idx).cuda()], dl[torch.from_numpy(idx).cuda()])
        assert np.float32(la).view(np.uint32) == lb.cpu().numpy().view(np.uint32)
    for x, y in zip(a.train_weights(), b.train_weights()):
        assert np.array_equal(bits(x), bits(y))


def test_begin_from_loaded_weights_and_the_weights_dir(tmp_path):
    for C in (15, 1):
        w = load_weights(C)[0] if C != 1 else tr.random_net(1, seed=1)
        lib.write_weights_dir(tmp_path, C, w)
        ctx = lib.Context(lib.default_params(channels=C))
        ctx.load_weights_dir(str(tmp_path) + "/")
        ctx.train_begin(lib.train_params())
        for x, y in zip(ctx.train_weights(), w):
            assert np.array_equal(bits(x), bits(np.asarray(y, F).ravel()))


def test_errors_leave_the_state_unchanged():
    C, relu = 3, 1
    w = tr.random_net(C, seed=2)
    images, labels = tr.random_images(8, C, seed=3), np.arange(8) % 2
    ctx = lib.Context(lib.default_params(channels=C, relu_after_conv=relu))
    with pytest.raises(lib.GpdbError, match=r"\[-3\]"):
        ctx.train_step(images, labels)
    with pytest.raises(lib.GpdbError, match=r"\[-3\]"):
        ctx.train_begin(lib.train_params())  # no loaded weights
    ctx.set_weights(w)
    scores0, _ = ctx.classify(images)
    ctx.train_begin(lib.train_params(optimizer="adam", lr=1e-3), init=w)
    ctx.train_step(images, labels)
    w1 = ctx.train_weights()
    ref = trainer(C, w, relu, optimizer="adam", lr=1e-3)
    ref.train_step(images, labels)
    for bad in ([2] + [0] * 7, [0] * 7 + [-1]):
        with pytest.raises(lib.GpdbError, match=r"\[-1\].*labels\["):
            ctx.train_step(images, bad)
    with pytest.raises(lib.GpdbError, match=r"\[-1\]"):
        ctx.train_step(images[:0], labels[:0])
    for bad in (lib.train_params(lr=-1.0), lib.train_params(lr=float("nan")), lib.train_params(optimizer="adam", betas=(1.0, 0.9))):
        with pytest.raises(lib.GpdbError, match=r"\[-1\]"):
            ctx.train_begin(bad)
    bad = lib.train_params()
    bad.optimizer = 7
    with pytest.raises(lib.GpdbError, match=r"\[-1\]"):
        ctx.train_begin(bad)
    for x, y in zip(ctx.train_weights(), w1):
        assert np.array_equal(bits(x), bits(y))
    # the optimiser state and step count survived too: the next step equals a context that never failed
    ctx.train_step(images, labels)
    ref.train_step(images, labels)
    for x, y in zip(ctx.train_weights(), ref.train_weights()):
        assert np.array_equal(bits(x), bits(y))
    # training never touched the classifier's weights
    assert np.array_equal(ctx.classify(images)[0], scores0)
    ctx.set_weights(ctx.train_weights())
    assert not np.array_equal(ctx.classify(images)[0], scores0)
    # an image size other than 60
    c48 = lib.Context(lib.default_params(channels=C, image_size=48))
    c48.train_begin(lib.train_params(), init=w)
    with pytest.raises(lib.GpdbError, match=r"\[-1\].*image_size 60"):
        c48.train_step(np.zeros((2, 48, 48, C), np.uint8), [0, 1])


CAMS4 = np.array([[0.0, 0.0, 0.0], [0.6, 0.0, 0.0], [-0.6, 0.0, 0.0], [0.0, 0.6, 0.0]])


def labelled_batch(C, n=64):
    """The INTEGRATION recipe on synthetic table views: candidates of one camera's view of each scene, labelled against
    four-camera ground truths of the same scenes; the first n / 2 positives and n / 2 negatives in candidate order."""
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
    pos, neg = (labels == 1).nonzero().flatten()[: n // 2], (labels == 0).nonzero().flatten()[: n // 2]
    assert len(pos) == len(neg) == n // 2, (len(pos), len(neg))
    sel = torch.cat([pos, neg])
    return images[sel].contiguous(), labels[sel].contiguous()


# Measured on an H100: both batches reach 100 % at the first check, after 10 steps. The run is deterministic; the budget
# allows one more check.
STEP_BUDGET = 20


@pytest.mark.parametrize("C", [15, 1])
def test_end_to_end_overfits_a_balanced_candidate_batch(C):
    import torch
    images, labels = labelled_batch(C)
    w, relu = load_weights(C)
    ctx = lib.Context(lib.default_params(channels=C, relu_after_conv=relu))
    ctx.train_begin(lib.train_params(optimizer="adam", lr=1e-4), init=w)
    for step in range(1, STEP_BUDGET + 1):
        ctx.train_step_tensors(images, labels)
        if step % 10 == 0:
            ctx.set_weights(ctx.train_weights())
            scores, _ = ctx.classify_tensors(images)
            acc = ((scores > 0).to(torch.int32) == labels).float().mean().item()
            if acc == 1.0:
                break
    print(f"C={C}: 100 % training accuracy after {step} steps")
    assert acc == 1.0
