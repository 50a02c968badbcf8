"""CPU tests that PIN the oracle (oracle/post_oracle.py, oracle/unet_oracle.py) to the reference:
  * against the golden fixtures in tests/golden/ (outputs of the unmodified reference, made by oracle/make_golden.py),
  * against the reference's only known-answer vector (src/postprocessing.py:95-111),
  * and against the reference's own functions on seeded inputs (tests/golden/live_reference.npz)."""
import os

import numpy as np
import pytest
import torch

from oracle import post_oracle as P
from oracle import synthetic
from oracle import unet_oracle as O

GOLD = os.path.join(os.path.dirname(__file__), "golden")


@pytest.fixture(scope="module")
def gp():
    return np.load(os.path.join(GOLD, "postproc.npz"))


@pytest.fixture(scope="module")
def gu():
    return np.load(os.path.join(GOLD, "unet.npz"))


def test_docstring_known_answer(gp):
    m = np.array([[0, 0, 1, 1], [1, 0, 0, 0], [1, 1, 1, 0], [0, 0, 1, 0]])
    want = np.array([[[1, 1, 0, 0], [0, 1, 1, 1], [0, 0, 0, 1], [2, 2, 0, 1]],
                     [[0, 0, 1, 1], [2, 0, 0, 0], [2, 2, 2, 0], [0, 0, 2, 0]]])
    got = P.label_multiclass_image(m)
    assert got.dtype == np.int32 and np.array_equal(got, want)
    assert np.array_equal(gp["docstring_labels"], want)


def test_postproc_oracle_matches_golden(gp):
    probs = gp["probs"]
    assert np.array_equal(probs, synthetic.probability_maps(3, 64, seed=1234, n_rect=12))
    for i, p in enumerate(probs):
        r = P.resize_image(p, (75, 75))
        assert r.dtype == np.float64 and np.array_equal(r, gp["resize_%d" % i])
        c = P.categorize_multilayer_image(r)
        assert c.dtype == bool and np.array_equal(c, gp["cat_%d" % i])
        l = P.label_multilayer_image(c)
        assert l.dtype == np.int32 and np.array_equal(l, gp["label_%d" % i])
        assert np.array_equal(P.dilate_image(l, 2), gp["dilate2_%d" % i])
        assert np.array_equal(P.dilate_image(l, 3), gp["dilate3_%d" % i])
        e = P.erode_image(c[1], 2)
        assert e.dtype == np.uint8 and np.array_equal(e, gp["erode2_%d" % i])
        assert np.array_equal(P.erode_image(c[1], 3), gp["erode3_%d" % i])
        _, s = P.build_score(gp["dilate2_%d" % i], r)
        assert np.allclose(np.array([float(v) for v in s[0]]), gp["score0_%d" % i], rtol=0, atol=0)
        assert np.allclose(np.array([float(v) for v in s[1]]), gp["score1_%d" % i], rtol=0, atol=0)
        assert np.array_equal(P.crop_image_center_per_class(p, 56, 56), gp["crop_%d" % i])
    assert np.array_equal(P.softmax(gp["softmax_in"], axis=1), gp["softmax_out"])


def test_resize_has_reference_zero_border(gp):
    """skimage<=0.17 + scipy 'constant' mode: output samples whose source coordinate falls outside the image are 0"""
    r = gp["resize_0"]
    assert (r[:, 0, :] == 0).all() and (r[:, -1, :] == 0).all() and (r[:, :, 0] == 0).all() and (r[:, :, -1] == 0).all()
    assert (r[:, 1:-1, 1:-1] > 0).all()


def test_unet_oracle_matches_golden(gu):
    x, t = synthetic.train_batch(2, 64, seed=1234, n_rect=6)
    assert np.array_equal(x, gu["x"]) and np.array_equal(t, gu["t"])
    sd = O.make_reference_like_state_dict(34, seed=1234)
    X, T = torch.from_numpy(x), torch.from_numpy(t)
    net = O.UNetOracle({k: v.clone() for k, v in sd.items()}, 34)
    with torch.no_grad():
        ev = net.forward(X, training=False)
    assert np.allclose(ev.numpy(), gu["eval_logits_34"], rtol=0, atol=1e-6)
    # training-mode forward, loss and gradients
    sd1 = {k: v.clone() for k, v in sd.items()}
    keys = O.trainable_keys(sd1)
    leaves = {k: sd1[k].clone().requires_grad_(True) for k in keys}
    work = dict(sd1)
    work.update(leaves)
    out = O.UNetOracle(work, 34).forward(X, training=True)
    assert np.allclose(out.detach().numpy(), gu["train_logits_34"], rtol=0, atol=1e-6)
    loss = O.mixed_loss(out, T, imsize=(256, 256))
    assert abs(float(loss) - float(gu["loss_34"])) < 1e-5 * abs(float(gu["loss_34"]))
    grads = dict(zip(keys, torch.autograd.grad(loss, [leaves[k] for k in keys], allow_unused=True)))
    for name in gu.files:
        if name.startswith("grad_34_"):
            k = name[len("grad_34_"):]
            ref = gu[name]
            assert np.allclose(grads[k].numpy(), ref, rtol=1e-3, atol=1e-6 * np.abs(ref).max() + 1e-12), k
    # closed-form loss gradient (what the CUDA kernel implements) == autograd
    lg = out.detach().clone().requires_grad_(True)
    l2 = O.mixed_loss(lg, T, imsize=(256, 256))
    l2.backward()
    l3, d3 = O.loss_and_dlogits_closed_form(out.detach(), T, imsize=(256, 256))
    assert abs(float(l3) - float(l2)) < 1e-5 * abs(float(l2))
    assert torch.allclose(d3, lg.grad, rtol=1e-4, atol=1e-9)


def test_train_step_oracle_matches_reference_fit_loop(gu):
    sd = O.make_reference_like_state_dict(34, seed=1234)
    X, T = torch.from_numpy(gu["x"]), torch.from_numpy(gu["t"])
    opt = O.AdamOracle(lr=5e-4, weight_decay=1e-4)
    loss, _, _ = O.train_step(sd, 34, X, T, opt, imsize=(256, 256))
    assert abs(float(loss) - float(gu["fit_loss_34"])) < 1e-5 * abs(float(gu["fit_loss_34"]))
    for name in gu.files:
        if name.startswith("step_34_"):
            k = name[len("step_34_"):]
            assert np.allclose(sd[k].numpy(), gu[name], rtol=1e-4, atol=1e-6), k
    loss2, _, _ = O.train_step(sd, 34, X, T, opt, imsize=(256, 256))
    assert abs(float(loss2) - float(gu["fit_loss2_34"])) < 2e-3 * abs(float(gu["fit_loss2_34"]))


def test_live_against_reference_code():
    """the reference's resize / categorize / label / dilate / erode and its network (state_dict of
    torch.manual_seed(7) + UNetResNet(34, ...), which make_reference_like_state_dict(34, seed=7) regenerates), stored by
    oracle/make_golden.py (live)"""
    g = np.load(os.path.join(GOLD, "live_reference.npz"))
    probs = synthetic.probability_maps(2, 48, seed=77, n_rect=8)
    for i, p in enumerate(probs):
        b = P.resize_image(p, (56, 56))
        assert np.array_equal(g["live_resize_%d" % i], b)
        c = g["live_cat_%d" % i]
        assert np.array_equal(c, P.categorize_multilayer_image(b))
        l = g["live_label_%d" % i]
        assert np.array_equal(l, P.label_multilayer_image(c))
        for k in (1, 2, 3, 4):
            assert np.array_equal(g["live_dilate%d_%d" % (k, i)], P.dilate_image(l, k))
            assert np.array_equal(g["live_erode%d_%d" % (k, i)], P.erode_image(c[1], k))
    # network: same state_dict -> identical logits
    sd = O.make_reference_like_state_dict(34, seed=7)
    x = torch.from_numpy(g["live_unet_x"])
    with torch.no_grad():
        got = O.UNetOracle(sd, 34).forward(x, training=False)
    assert torch.equal(torch.from_numpy(g["live_unet_logits"]), got)


@pytest.mark.parametrize("case", [0, 1, 2])
def test_unet_oracle_matches_config_goldens(case):
    """tests/golden/unet_configs_*.npz (BASELINE.json configs 1 / 2 / 5: R34 b2 @256, R101 @320, R152 @512) was produced
    by the UNMODIFIED reference from seed 1234; the seed-regenerated weights + inputs and the oracle network must reproduce
    its eval logits (image 0), which pins both the fixture's inputs and the oracle at those depths / resolutions."""
    from oracle.make_golden_cases import CONFIG_CASES, LOGIT_STRIDE, load_unet_golden
    tag, enc, depth, n, s = CONFIG_CASES[case]
    g = load_unet_golden("configs")
    sd = O.make_reference_like_state_dict(depth, seed=1234)
    x, _ = synthetic.train_batch(n, s, seed=1234)
    with torch.no_grad():
        ev = O.UNetOracle(sd, depth).forward(torch.from_numpy(x[:1]), training=False)[:, :, ::LOGIT_STRIDE, ::LOGIT_STRIDE]
    ref = g["eval_logits_" + tag]
    assert ev.shape == ref.shape
    assert np.abs(ev.numpy() - ref).max() < 1e-6
