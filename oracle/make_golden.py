"""TEST INFRASTRUCTURE — generates tests/golden/*.npz by running the UNMODIFIED reference (a checkout of
neptune-ai/open-solution-mapping-challenge at MCB_REFERENCE_ROOT, imported through oracle/ref_shim.py) on seeded
synthetic inputs:  python -m oracle.make_golden [postproc|unet|configs|conditioned|live ...]
The fixtures pin the CPU oracle restatements (oracle/post_oracle.py, oracle/unet_oracle.py); the GPU tests then compare
the CUDA path with the oracle and with these fixtures."""
import json
import os
import sys
import warnings

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_shim, synthetic  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")


def golden_postproc(pp, ut):
    probs = synthetic.probability_maps(3, 64, seed=1234, n_rect=12)
    rec = {"probs": probs}
    for i, p in enumerate(probs):
        r = pp.resize_image(p, (75, 75))
        c = pp.categorize_multilayer_image(r)
        l = pp.label_multilayer_image(c)
        d = pp.dilate_image(l, 2)
        d3 = pp.dilate_image(l, 3)
        e = pp.erode_image(c[1], 2)          # 2-D branch (the multi-layer branch of the reference is broken)
        e3 = pp.erode_image(c[1], 3)
        _, s = pp.build_score(d, r)
        crop = pp.crop_image_center_per_class(p, 56, 56)
        rec.update({"resize_%d" % i: r, "cat_%d" % i: c, "label_%d" % i: l, "dilate2_%d" % i: d, "dilate3_%d" % i: d3,
                    "erode2_%d" % i: e, "erode3_%d" % i: e3, "crop_%d" % i: crop,
                    "score0_%d" % i: np.array([float(v) for v in s[0]]),
                    "score1_%d" % i: np.array([float(v) for v in s[1]])})
    logits = np.random.RandomState(5).randn(2, 2, 16, 16).astype(np.float32) * 3
    rec["softmax_in"] = logits
    rec["softmax_out"] = ut.softmax(logits, axis=1)
    m = np.array([[0, 0, 1, 1], [1, 0, 0, 0], [1, 1, 1, 0], [0, 0, 1, 0]])
    rec["docstring_mask"] = m
    rec["docstring_labels"] = pp.label_multiclass_image(m)
    np.savez_compressed(os.path.join(OUT, "postproc.npz"), **rec)
    print("postproc.npz", len(rec), "arrays")


def golden_unet(um, mo):
    rec = {}
    for depth, enc in ((34, "ResNet34"),):
        cfg = ref_shim.reference_unet_config(enc)
        torch.manual_seed(1234)
        model = mo.PyTorchUNetWeighted(**cfg)   # builds UNetResNet(depth) + Adam(lr 5e-4, wd 1e-4) like the reference
        x, t = synthetic.train_batch(2, 64, seed=1234, n_rect=6)
        X, T = torch.from_numpy(x), torch.from_numpy(t)
        model.model.eval()
        with torch.no_grad():
            rec["eval_logits_%d" % depth] = model.model(X).numpy()
        model.model.train()
        # loss + gradients of the first step (without the update)
        out = model.model(X)
        name, loss_fn, weight = model.loss_function[0]
        loss = loss_fn(out, T) * weight
        loss.backward()
        rec["train_logits_%d" % depth] = out.detach().numpy()
        rec["loss_%d" % depth] = np.array(float(loss))
        sd = dict(model.model.named_parameters())
        for k in ("final.weight", "final.bias", "dec0.conv.weight", "dec1.block.1.weight", "center.block.0.conv.bias",
                  "encoder.layer1.0.conv1.weight", "encoder.bn1.weight", "encoder.conv1.weight"):
            rec["grad_%d_%s" % (depth, k)] = sd[k].grad.detach().numpy().copy()
        # undo the forward's running-stat update, then run the reference's own train step
        torch.manual_seed(1234)
        model = mo.PyTorchUNetWeighted(**cfg)
        res = model._fit_loop([X, T])
        rec["fit_loss_%d" % depth] = np.array(float(res["sum"]))
        sd2 = model.model.state_dict()
        for k in ("final.weight", "dec0.conv.bias", "encoder.bn1.running_mean", "encoder.bn1.running_var",
                  "encoder.layer4.2.bn2.weight", "center.block.1.bias"):
            rec["step_%d_%s" % (depth, k)] = sd2[k].numpy().copy()
        res2 = model._fit_loop([X, T])
        rec["fit_loss2_%d" % depth] = np.array(float(res2["sum"]))
    rec["x"], rec["t"] = x, t
    np.savez_compressed(os.path.join(OUT, "unet.npz"), **rec)
    print("unet.npz", {k: v.shape for k, v in rec.items() if v.ndim == 0 or "logits" in k})


from oracle.make_golden_cases import CONFIG_CASES, CONFIG_GRAD_KEYS, GRAD_HEAD, LOGIT_STRIDE, save_unet_golden  # noqa: E402


def golden_unet_configs(um, mo):
    """reference logits (eval + train), loss and a spread of gradients at the BASELINE.json configurations.  Inputs
    and the initial weights are NOT stored: both sides regenerate them from the seed (synthetic.train_batch(n, s, 1234),
    unet_oracle.make_reference_like_state_dict(depth, seed=1234), which test_oracle_pins pins to the reference's own
    initialisation)."""
    rec = {}
    for tag, enc, depth, n, s in CONFIG_CASES:
        cfg = ref_shim.reference_unet_config(enc, image_hw=(256, 256))
        torch.manual_seed(1234)
        model = mo.PyTorchUNetWeighted(**cfg)
        x, t = synthetic.train_batch(n, s, seed=1234)
        X, T = torch.from_numpy(x), torch.from_numpy(t)
        model.model.eval()
        with torch.no_grad():
            # eval mode is per image: image 0 is enough
            rec["eval_logits_" + tag] = model.model(X[:1]).numpy()[:, :, ::LOGIT_STRIDE, ::LOGIT_STRIDE].copy()
        model.model.train()
        out = model.model(X)
        name, loss_fn, weight = model.loss_function[0]
        loss = loss_fn(out, T) * weight
        loss.backward()
        rec["train_logits_" + tag] = out.detach().numpy()[:, :, ::LOGIT_STRIDE, ::LOGIT_STRIDE].copy()
        rec["loss_" + tag] = np.array(float(loss))
        sd = dict(model.model.named_parameters())
        for k in CONFIG_GRAD_KEYS:
            rec["grad_%s_%s" % (tag, k)] = sd[k].grad.detach().numpy().reshape(-1)[:GRAD_HEAD].copy()
        print(tag, "loss", float(loss), "logit range", float(out.min()), float(out.max()), flush=True)
    save_unet_golden("configs", rec)


def golden_unet_conditioned(um, mo):
    """the same configurations on the conditioned checkpoint (damped residual branches, calibrated running statistics):
    the regime of a trained net, where logits AND deep-encoder gradients are reproducible quantities.  The checkpoint
    is regenerated from the seed on both sides (oracle.unet_oracle.conditioned_state_dict); here it is loaded into the
    UNMODIFIED reference network, whose own calibration pass must reproduce the checkpoint's running statistics."""
    from oracle import unet_oracle as O
    rec = {}
    s3 = LOGIT_STRIDE
    for tag, enc, depth, n, s in CONFIG_CASES:
        x, t = synthetic.train_batch(n, s, seed=1234)
        X, T = torch.from_numpy(x), torch.from_numpy(t)
        sd = O.conditioned_state_dict(depth, X, seed=1234)
        cfg = ref_shim.reference_unet_config(enc, image_hw=(256, 256))
        model = mo.PyTorchUNetWeighted(**cfg)
        net = model.model
        raw = O.make_reference_like_state_dict(depth, seed=1234)
        last = "bn2" if depth == 34 else "bn3"
        for k in raw:   # damp, then let the reference calibrate itself (momentum 1): must equal the oracle's checkpoint
            if k.startswith("encoder.layer") and k.endswith("." + last + ".weight"):
                raw[k] = raw[k] * 0.25
        for k in list(raw):
            for new, old in (("conv2.", "encoder.layer1."), ("conv3.", "encoder.layer2."), ("conv4.", "encoder.layer3."),
                             ("conv5.", "encoder.layer4.")):
                if k.startswith(new):
                    raw[k] = raw[old + k[len(new):]]
        net.load_state_dict(raw)
        bns = [m for m in net.modules() if isinstance(m, torch.nn.BatchNorm2d)]
        for m in bns:
            m.momentum = 1.0
        net.train()
        with torch.no_grad():
            net(X)
        for m in bns:
            m.momentum = 0.1
        got = net.state_dict()
        for k, v in sd.items():
            if v.is_floating_point():
                assert torch.equal(got[k], v), ("reference calibration differs from the oracle checkpoint", k)
        net.eval()
        with torch.no_grad():
            rec["eval_logits_" + tag] = net(X[:1]).numpy()[:, :, ::s3, ::s3].copy()
        net.train()
        out = net(X)
        name, loss_fn, weight = model.loss_function[0]
        loss = loss_fn(out, T) * weight
        loss.backward()
        rec["train_logits_" + tag] = out.detach().numpy()[:, :, ::s3, ::s3].copy()
        rec["loss_" + tag] = np.array(float(loss))
        params = dict(net.named_parameters())
        for k in CONFIG_GRAD_KEYS:
            rec["grad_%s_%s" % (tag, k)] = params[k].grad.detach().numpy().reshape(-1)[:GRAD_HEAD].copy()
        print(tag, "conditioned: loss", float(loss), "logit range", float(out.min()), float(out.max()),
              "eval range", float(rec["eval_logits_" + tag].min()), float(rec["eval_logits_" + tag].max()), flush=True)
    save_unet_golden("conditioned", rec)


def golden_live(um, mo, pp, ut):
    """what the CPU pins (tests/test_oracle_pins.py, test_input_cpu.py, test_instances_cpu.py) compare the oracles
    against: the reference's own post-processing, network, preparation and test-time-augmentation functions on the
    seeded inputs those tests regenerate"""
    ref_shim.install()
    import src.loaders as lo
    import src.preparation as prep
    from oracle import instances_oracle as I
    rec = {}
    for i, p in enumerate(synthetic.probability_maps(2, 48, seed=77, n_rect=8)):
        a = pp.resize_image(p, (56, 56))
        c = pp.categorize_multilayer_image(a)
        l = pp.label_multilayer_image(c)
        rec["live_resize_%d" % i], rec["live_cat_%d" % i], rec["live_label_%d" % i] = a, c, l
        for k in (1, 2, 3, 4):
            rec["live_dilate%d_%d" % (k, i)] = pp.dilate_image(l, k)
            rec["live_erode%d_%d" % (k, i)] = pp.erode_image(c[1], k)
    torch.manual_seed(7)
    ref = um.UNetResNet(34, 2, 32, 0.0, False, True)   # = unet_oracle.make_reference_like_state_dict(34, seed=7)
    x = torch.randn(1, 3, 64, 64)
    ref.eval()
    with torch.no_grad():
        rec["live_unet_x"], rec["live_unet_logits"] = x.numpy(), ref(x).numpy()
    # src/preparation.py: distances to the two nearest objects, size matrix
    rs = np.random.RandomState(1)
    masks = np.stack([synthetic.rectangles_mask(rs, 40, 52, n_rect=1, lo=4, hi=10)[0] for _ in range(5)])
    d = np.zeros((40, 52))
    for m in masks:
        d = prep.update_distances(d, m)
    rec["prep_dist_sum"], rec["prep_dist_second"] = prep.clean_distances(d.copy())
    rec["prep_size_matrix"] = prep.get_size_matrix((masks.sum(0) > 0).astype(np.uint8))
    # src/loaders.py: test-time augmentation generator / transform / inverse / aggregation; NMS
    specs = I.tta_specs()
    gen = lo.TestTimeAugmentationGenerator(flip_ud=True, flip_lr=True, rotation=True, color_shift_runs=False)
    got = gen.transform(np.array([["a"], ["b"]], dtype=object))
    rec["tta_params_json"] = np.array(json.dumps(got["tta_params"]))
    rec["tta_img_ids"] = np.array(got["img_ids"])
    rs = np.random.RandomState(5)
    img = rs.randint(0, 255, (12, 12, 3)).astype(np.uint8)
    fwd, inv, preds = [], [], []
    for p in specs:
        fwd.append(np.asarray(lo.test_time_augmentation_transform(img, p)))
        pr = rs.rand(2, 12, 12).astype(np.float32)
        inv.append(lo.test_time_augmentation_inverse_transform(pr, p))
        preds.append(pr)
    rec["tta_forward"], rec["tta_inverse"] = np.stack(fwd), np.stack(inv)
    for method in ("gmean", "mean", "max", "min"):
        agg = lo.TestTimeAugmentationAggregator(method, 2).transform(preds * 2, specs * 2, [0] * 16 + [1] * 16)
        rec["tta_agg_" + method] = np.stack(agg["aggregated_prediction"])
    lab = np.zeros((2, 20, 20), np.int32)
    lab[0, 2:8, 2:8] = 1
    lab[0, 10:18, 10:18] = 2
    lab[1, 3:8, 2:8] = 1
    lab[1, 12:14, 12:14] = 2
    rec["nms_scores"] = np.array(pp.remove_overlapping_masks(lab, [[0.9, 0.5], [0.8, 0.7]], 0.5)[1])
    np.savez_compressed(os.path.join(OUT, "live_reference.npz"), **rec)
    print("live_reference.npz", os.path.getsize(os.path.join(OUT, "live_reference.npz")) >> 10, "KiB")


if __name__ == "__main__":
    warnings.filterwarnings("ignore")
    os.makedirs(OUT, exist_ok=True)
    um, mo, pp, ut = ref_shim.reference_modules()
    which = sys.argv[1:] or ["postproc", "unet", "configs", "conditioned", "live"]
    if "postproc" in which:
        golden_postproc(pp, ut)
    if "unet" in which:
        golden_unet(um, mo)
    if "configs" in which:
        golden_unet_configs(um, mo)
    if "conditioned" in which:
        golden_unet_conditioned(um, mo)
    if "live" in which:
        golden_live(um, mo, pp, ut)
