"""The ResNet101 U-Net train step (320x320, built as oracle.step_checks.BenchStep builds it) across what a training run
does between steps, bit for bit.  The reference trains at batch 20, and its callbacks act between steps:
ExponentialLRScheduler steps a torch ExponentialLR on the transformer's optimizer; ModelCheckpoint's save_model runs
model.eval(); model.cpu(); torch.save(model.state_dict()); model.cuda(); model.train(), which re-creates the arenas
and forces every train step to be captured again (Model._fused_step, AdamState.rebind); the validation monitor runs eval
forwards of the same net, which write the bf16 operand arena the captured train steps read (refresh_operands).

Every cross-CTA sum of the step is added in a fixed order, so each test compares two runs from the same weights and
batches: loss, logits, gradients, fp32 weights, Adam moments, the bf16 operand copy and the running statistics, bitwise
(oracle.step_checks.snapshot_mismatches).
  1. learning-rate changes reach the captured Adam: ExponentialLR (gamma 0.9) stepped after every batch for 10 steps,
     more than the 8 slots of FusedTrainStep._hyper_ring, then a plateau-style cut (x 0.3) written into the param
     group: every step is exactly whole-arena Adam of its own gradients with the lr the optimizer held and the t it
     ran at.  Changing betas, eps or weight_decay after capture raises and leaves the step count and the state alone;
  2. a checkpoint round trip between steps 2 and 3 changes no step; the saved file equals the uninterrupted run's
     state_dict() after step 2, key for key (with the `module.` prefix) and bit for bit; Model.load() of it gives the
     same eval forward, and the same next train step in a model whose captured step read other weights before;
  3. validation passes (ValidationMonitorSegmentation with validate_with_map, 45 tiles at batch 20: 20, 20, 5) after
     steps 2 and 4 change no step; their eval forwards equal a separately built eval plan's, and their AP equals the
     COCOeval oracle chain (oracle.coco_oracle) on that plan's logits;
  4. fit() for up to 4 epochs of 47 tiles at batch 20 (20, 20, 7) with stand-ins of the reference's callbacks
     (per-epoch ExponentialLR, checkpoint on AP improvement through save_model, the device validation monitor,
     early stopping on the validation AP with patience 0) equals a hand-driven loop of _fit_loop calls that runs
     first, sets the lr each epoch and makes save_model's round trip after epochs 0 and 1.  The ground truth is every
     other detection of the hand-driven loop's epoch 1, through a separate eval plan, so the AP rules must save after
     epochs 0 and 1 and stop after epoch 2: fit() must give the oracle's APs, those checkpoints and that stop, the
     same losses and epoch-end states, and epoch 1's state on disk.  The callbacks run in the reference's order, and
     the datagen's `steps` ends every epoch as `if batch_id == steps: break` does.
At most one ResNet101 model is alive at a time (test 4 asserts it between its phases); what is compared across runs is
kept on the host.

Measured on an H100 80GB HBM3 at its 700 W power limit: the file takes about 125 s.
  1. 21 s, peak 8.8 GiB: 13 steps checked against Adam, 3 refused changes;
  2. 28 s, 14.8 GiB: 5 + 5 steps compared, 1 checkpoint file, 1 eval forward after load(), 1 train step after load();
  3. 31 s, 10.5 GiB: 5 + 5 steps compared, 6 validation batches bitwise, 2 APs.  The ground truth is every other
     detection after step 2 (180 detections), so the first AP is 0.4824, equal to the oracle's; after step 4 the net's
     45 detections match none of it, and both give 0;
  4. 31 s, 33.5 GiB (one model, with train plans at 20 and 7, eval plans at 20 and 5, and two round trips): 9 losses,
     3 epoch-end states, 3 APs and 1 checkpoint file compared.  The epochs give 45, 0 and 0 detections, so the ground
     truth from epoch 1 is empty and the APs are -1 (COCOeval's value with detections and no ground truth), 0 and 0
     (no detections): the improvement at epoch 1 saves the checkpoint that a keep-the-first or keep-the-last rule, or
     a monitor that returns one constant AP, would not.
Deliberate mutations, each caught: the Adam scalars computed once at capture (1 and 2); m and v zeroed in
AdamState.rebind (2); refresh_operands() skipped in Model.load (2); an eval forward that writes the bf16 operand copy
from a stale fp32 copy (3; 2 and 4 do not see it: 2 runs its eval forward in both of its runs, and in 4 every
validation that a train step follows is followed by a round trip, whose re-capture refreshes the operand copy);
fit() breaking one batch after `steps` (4); a monitor that returns the first epoch's AP (4).  Test 4 shares the
train step, AdamState.rebind and save_model with its hand-driven loop, so the first two mutations change both of its
runs alike: tests 1 and 2 are the ones that catch them."""
import json
import os
import types

import numpy as np
import pytest
import torch
from torch import nn

from oracle import coco_oracle as CO
from oracle import instances_oracle as I
from oracle import post_oracle as P
from oracle.step_checks import (SEED, BenchStep, adam_mismatches, arena_layout, batch, free_device_memory, host,
                                same_bits, seeded_sd, snapshot, snapshot_mismatches)
from oracle.step_checks import rng_and_peak_memory  # noqa: F401  (fixture)

# the fused step runs Adam itself, never optimizer.step(), which torch's schedulers warn about
pytestmark = [pytest.mark.gpu, pytest.mark.filterwarnings("ignore:Detected call of `lr_scheduler.step:UserWarning")]

ENCODER = "ResNet101"
N_TRAIN = 20              # neptune.yaml's batch_size_train
EPOCH_TILES = 47          # 20 + 20 + 7
N_VAL = 45                # 20 + 20 + 5
SMALL = 14                # small_annotations_size
IMAGE_IDS = list(range(700, 700 + N_VAL))


# ---------------------------------------------------------------------------------------------------------------------
# helpers
# ---------------------------------------------------------------------------------------------------------------------
def train_batches(seed, tiles=EPOCH_TILES, n=N_TRAIN):
    """an epoch of `tiles` host tiles as the DataLoader hands them over: batches of n and the partial rest"""
    x, t = batch(seed, tiles)
    return [(x[i:i + n], t[i:i + n]) for i in range(0, tiles, n)]


def val_batches():
    x, _ = batch(SEED + 500, N_VAL)
    return [x[i:i + N_TRAIN] for i in range(0, N_VAL, N_TRAIN)]


def wrap(run, cuda):
    """fit()'s DataParallel wrapper around the net, so that state_dict() carries the `module.` prefix"""
    run.model.model = nn.DataParallel(run.model.model, device_ids=[cuda.index or 0])
    return run.model.model


def save_model(model, path):
    """the reference's save_model (src/steps/pytorch/utils.py) on a device"""
    model.eval()
    model.cpu()
    torch.save(model.state_dict(), path)
    model.cuda()
    model.train()


def host_state(model):
    return {k: host(v) for k, v in model.state_dict().items()}


def state_mismatches(a, b):
    """differences between two state dicts, key for key (order included) and bit for bit"""
    if list(a) != list(b):
        return ["keys differ: %s" % (sorted(set(a) ^ set(b))[:5] or "the same keys in another order")]
    out = []
    for k in a:
        x, y = a[k], b[k]
        ok = x.shape == y.shape and x.dtype == y.dtype and (same_bits(x, y) if x.is_floating_point() else torch.equal(x, y))
        if not ok:
            out.append(k)
    return out


def eval_logits(model, xs, cuda):
    """the eval forward of `model` (the wrapper or the net) on host batches -> host logits"""
    model.eval()
    with torch.no_grad():
        out = [host(model(x.to(cuda))) for x in xs]
    model.train()
    return out


def state_of(model, loss):
    """snapshot of the transformer's last train step"""
    return snapshot(types.SimpleNamespace(net=model._net(), fused=model._fused), loss)


class EvalPlan:
    """a separately built eval model: load a state dict, run the eval forward on the validation tiles"""

    def __init__(self):
        from mcb200.models import PyTorchUNet
        import bench
        self.model = PyTorchUNet(**bench.unet_config(ENCODER))

    def logits(self, sd, cuda):
        net = self.model.model
        net.load_state_dict({(k[7:] if k.startswith("module.") else k): v for k, v in sd.items()})
        self.model._to_device()
        return eval_logits(net, val_batches(), cuda)


def oracle_results(logits, monkeypatch):
    """the reference's validation chain on host logits: softmax, resize to 300x300, argmax, label, build_score,
    create_annotations"""
    from mcb200 import ops
    probs = np.concatenate([ops.softmax2(l.cuda().contiguous()).cpu().numpy() for l in logits])
    preds = []
    for p in probs:
        r = P.resize_image(p, (300, 300))
        preds.append(P.build_score(P.label_multiclass_image(P.categorize_image(r)), r))
    monkeypatch.setattr(I, "rle_encode", CO.rle_encode)
    return I.create_annotations(IMAGE_IDS, preds, [None, 100], [1, 1])


def write_ground_truth(results, data_dir):
    """every other detection is a ground-truth instance, some of them crowds"""
    anns = []
    for j, a in enumerate(results[::2]):
        anns.append({"id": j + 1, "image_id": a["image_id"], "category_id": 100, "iscrowd": int(j % 7 == 3),
                     "area": CO.area(a["segmentation"]), "segmentation": dict(a["segmentation"])})
    gt = {"images": [{"id": i, "height": 300, "width": 300} for i in IMAGE_IDS], "annotations": anns,
          "categories": [{"id": 100}]}
    os.makedirs(os.path.join(data_dir, "val"), exist_ok=True)
    with open(os.path.join(data_dir, "val", "annotation.json"), "w") as f:
        json.dump(gt, f)
    return gt


def oracle_ap(gt, results):
    c_gt = CO.COCO()
    c_gt.dataset = json.loads(json.dumps(gt))
    c_gt.createIndex()
    ev = CO.COCOevalOracle(c_gt, c_gt.loadRes(json.loads(json.dumps(results))), np.asarray(IMAGE_IDS), [100], SMALL)
    ev.evaluate()
    ev.accumulate()
    ev.summarize()
    return float(ev.stats[0])


def monitor(data_dir, record=None):
    """the device validation monitor; `record` collects the host logits of its eval forwards"""
    from mcb200.callbacks import ValidationMonitorSegmentation
    mon = ValidationMonitorSegmentation(data_dir=data_dir, small_annotations_size=SMALL, validate_with_map=True,
                                        epoch_every=1)
    if record is not None:
        add = mon.add_logits

        def add_logits(logits, image_ids):
            record.append(host(logits))
            return add(logits, image_ids)
        mon.add_logits = add_logits
    return mon


def compare_runs(layout, a, b, what):
    for i, (x, y) in enumerate(zip(a, b)):
        bad = snapshot_mismatches(layout, x, y)
        print("%s, step %d: loss %.7f, equal: %s" % (what, i + 1, float(x["loss"]), not bad))
        assert not bad, "%s, step %d: %s" % (what, i + 1, "; ".join(bad))
    assert len(a) == len(b)


# ---------------------------------------------------------------------------------------------------------------------
# 1. learning-rate changes
# ---------------------------------------------------------------------------------------------------------------------
def test_learning_rate_changes_reach_the_captured_adam(mcb, cuda):
    run = BenchStep(ENCODER, seeded_sd(ENCODER), cuda, N_TRAIN)
    layout = arena_layout(run.net)
    opt = run.model.optimizer
    sched = torch.optim.lr_scheduler.ExponentialLR(opt, gamma=0.9)
    lrs = []
    for i in range(12):
        if i == 11:
            opt.param_groups[0]["lr"] *= 0.3            # a plateau-style cut written into the param group
        X, T = (t.to(cuda) for t in batch(SEED + 40 + i, N_TRAIN))
        lrs.append(run.lr())
        replay = run.is_replay(X, T)
        _, bad = adam_mismatches(run, layout, X, T)
        print("step %2d (%s), lr %.6e: fused Adam == Adam with this lr and t: %s" % (
            i + 1, "graph replay" if replay else "eager", lrs[-1], not bad))
        assert not bad, "step %d, lr %r: %s" % (i + 1, lrs[-1], "; ".join(bad))
        if i < 10:
            sched.step()
    assert len(set(lrs)) == len(lrs) and lrs[11] == lrs[10] * 0.3, lrs

    # betas, eps and weight decay are baked into the captured launches: changing them is refused before the step
    # counts, and the next step with the settings restored is the next t
    g = opt.param_groups[0]
    X, T = (t.to(cuda) for t in batch(SEED + 60, N_TRAIN))
    for key, value in (("betas", (0.8, 0.999)), ("eps", 1e-6), ("weight_decay", 0.0)):
        saved, t0, p = g[key], run.fused.opt.t, host(run.net._p32)
        g[key] = value
        with pytest.raises(RuntimeError, match="changed after the train step was captured"):
            run.step(X, T)
        g[key] = saved
        assert run.fused.opt.t == t0, "a refused step must not count: t %d, was %d" % (run.fused.opt.t, t0)
        assert same_bits(host(run.net._p32), p)
    _, bad = adam_mismatches(run, layout, X, T)
    assert not bad, "the step after the refused ones: %s" % "; ".join(bad)
    assert run.fused.opt.t == 13
    del run, opt, sched
    free_device_memory()


# ---------------------------------------------------------------------------------------------------------------------
# 2. checkpoint round trip
# ---------------------------------------------------------------------------------------------------------------------
def test_checkpoint_round_trip_between_steps_changes_nothing(mcb, cuda, tmp_path):
    import bench
    from mcb200.models import PyTorchUNetWeighted
    sd = seeded_sd(ENCODER)
    batches = [tuple(t.to(cuda) for t in batch(SEED + 70 + i, N_TRAIN)) for i in range(5)]
    xv = val_batches()[:1]
    path = str(tmp_path / "checkpoint.torch")

    # B: five steps; its state dict and eval forward after step 2 are what the checkpoint must hold and give
    run = BenchStep(ENCODER, sd, cuda, N_TRAIN)
    model = wrap(run, cuda)
    layout = arena_layout(run.net)
    b_steps = []
    for i, (X, T) in enumerate(batches):
        b_steps.append(snapshot(run, run.step(X, T)))
        if i == 1:
            b_state = host_state(model)
            b_eval = eval_logits(model, xv, cuda)
    del run, model
    free_device_memory()

    # A: the same five steps with save_model between steps 2 and 3
    run = BenchStep(ENCODER, sd, cuda, N_TRAIN)
    model = wrap(run, cuda)
    a_steps = []
    for i, (X, T) in enumerate(batches):
        a_steps.append(snapshot(run, run.step(X, T)))
        if i == 1:
            a_eval = eval_logits(model, xv, cuda)
            gen = run.net._generation
            save_model(model, path)
            assert run.net._generation > gen and run.net._p32.is_cuda
    assert run.model._opt_state.t == 5 and run.fused.graphs is not None
    del run, model
    free_device_memory()
    compare_runs(layout, b_steps, a_steps, "round trip after step 2 against none")
    assert same_bits(a_eval[0], b_eval[0])

    saved = torch.load(path, map_location="cpu")
    assert all(k.startswith("module.") for k in saved)
    bad = state_mismatches(b_state, saved)
    assert not bad, "the checkpoint differs from the state after step 2: %s" % bad[:10]

    # Model.load() into a fresh model: the eval forward of the loaded weights
    model = PyTorchUNetWeighted(**bench.unet_config(ENCODER))
    model.load(path)
    got = eval_logits(model._net(), xv, cuda)
    assert same_bits(got[0], b_eval[0]), "eval forward after load(): %d logits differ" % int(
        (got[0] != b_eval[0]).sum())
    del model, got
    free_device_memory()

    # Model.load() in the middle of training: the captured step must read the loaded weights
    run = BenchStep(ENCODER, sd, cuda, N_TRAIN)
    run.step(*(t.to(cuda) for t in batch(SEED + 80, N_TRAIN)))
    run.model.load(path)
    c = snapshot(run, run.step(*batches[2]))
    assert run.fused.graphs is not None
    b = b_steps[2]
    assert same_bits(c["loss"], b["loss"]), "loss after load(): %r, uninterrupted run %r" % (c["loss"], b["loss"])
    assert same_bits(c["logits"], b["logits"]), "logits after load()"
    assert not [k for k in b["stats"] if not same_bits(b["stats"][k], c["stats"][k])], "running statistics"
    del run
    free_device_memory()


# ---------------------------------------------------------------------------------------------------------------------
# 3. validation between steps
# ---------------------------------------------------------------------------------------------------------------------
def test_validation_between_steps_changes_nothing(mcb, cuda, tmp_path, monkeypatch):
    import pandas as pd
    sd = seeded_sd(ENCODER)
    batches = [tuple(t.to(cuda) for t in batch(SEED + 90 + i, N_TRAIN)) for i in range(5)]

    # B: five steps without validation; the state dicts after steps 2 and 4 for the eval plan
    run = BenchStep(ENCODER, sd, cuda, N_TRAIN)
    model = wrap(run, cuda)
    layout = arena_layout(run.net)
    b_steps, states = [], []
    for i, (X, T) in enumerate(batches):
        b_steps.append(snapshot(run, run.step(X, T)))
        if i in (1, 3):
            states.append(host_state(model))
    del run, model
    free_device_memory()

    # a separately built eval plan at those weights, the oracle chain on its logits, the ground truth from step 2's
    ev = EvalPlan()
    plan_logits = [ev.logits(s, cuda) for s in states]
    del ev
    free_device_memory()
    results = [oracle_results(lg, monkeypatch) for lg in plan_logits]
    print("detections after steps 2 and 4: %d, %d" % tuple(len(r) for r in results))
    data_dir = str(tmp_path)
    gt = write_ground_truth(results[0], data_dir)
    want = [oracle_ap(gt, r) if r else 0.0 for r in results]     # no detections: 0, as the monitor rules

    # A: the same steps with the validation monitor after steps 2 and 4
    run = BenchStep(ENCODER, sd, cuda, N_TRAIN)
    model = wrap(run, cuda)
    seen = []
    mon = monitor(data_dir, seen)
    transformer = types.SimpleNamespace(model=model, optimizer=run.model.optimizer, loss_function=None,
                                        output_names=["multichannel_map"], validation_loss={})
    mon.set_params(transformer, validation_datagen=(val_batches(), None), meta_valid=pd.DataFrame({"ImageId": IMAGE_IDS}))
    mon.on_train_begin()
    a_steps = []
    for i, (X, T) in enumerate(batches):
        a_steps.append(snapshot(run, run.step(X, T)))
        if i in (1, 3):
            mon.on_epoch_end()
    assert run.net.training
    transformer.model = transformer.optimizer = None
    del run, model, mon
    free_device_memory()
    compare_runs(layout, b_steps, a_steps, "validation after steps 2 and 4 against none")

    assert len(seen) == 6 and [l.shape[0] for l in seen] == [20, 20, 5] * 2
    for e in range(2):
        for j in range(3):
            assert same_bits(seen[3 * e + j], plan_logits[e][j]), \
                "validation %d, batch %d: the monitor's eval forward differs from the eval plan's" % (e + 1, j + 1)
        got = transformer.validation_loss[e]["sum"]
        print("validation %d: AP %.6f, oracle %.6f" % (e + 1, float(got[0]), want[e]))
        assert got.shape == (1,) and got.item() == torch.tensor([want[e]], dtype=torch.float32).item()


# ---------------------------------------------------------------------------------------------------------------------
# 4. fit() end to end
# ---------------------------------------------------------------------------------------------------------------------
class Loader:
    """a re-iterable DataLoader stand-in: epoch e's batches, then one more batch that the datagen's `steps` leaves
    unread.  Records what is drawn"""

    def __init__(self, epochs, extra):
        self.epochs, self.extra, self.epoch, self.drawn = epochs, extra, -1, []

    def __iter__(self):
        self.epoch += 1
        for i, b in enumerate(self.epochs[self.epoch] + [self.extra]):
            self.drawn.append((self.epoch, i))
            yield list(b)


class Callback:
    """the part of the reference's Callback these stand-ins use: the transformer's model, optimizer and
    validation_loss, the epoch counter, and a shared event log"""

    def __init__(self, log):
        self.log = log

    def set_params(self, transformer, validation_datagen=None, meta_valid=None):
        self.transformer, self.model, self.optimizer = transformer, transformer.model, transformer.optimizer
        self.validation_loss = transformer.validation_loss

    def on_train_begin(self):
        self.epoch_id = 0

    def on_train_end(self): pass
    def on_epoch_begin(self): pass
    def on_batch_begin(self): pass
    def on_batch_end(self, metrics=None): pass
    def training_break(self): return False

    def ap(self):
        """the epoch's validation AP, read between model.eval() and model.train() as the reference's callbacks do"""
        self.model.eval()
        ap = float(self.validation_loss[self.epoch_id]["sum"].data.cpu().numpy()[0])
        self.model.train()
        return ap


class Snapshots(Callback):
    """the training state after every batch's loss and at every epoch end (first in the list: before validation)"""

    def on_train_begin(self):
        super().on_train_begin()
        self.losses, self.epochs = [], []

    def on_batch_end(self, metrics=None):
        self.losses.append(host(metrics["sum"]))

    def on_epoch_end(self):
        self.log.append(("snapshot", self.epoch_id))
        self.epochs.append(state_of(self.transformer, self.losses[-1]))
        self.epoch_id += 1


class Validation(Callback):
    """the device validation monitor, logged"""

    def __init__(self, log, mon):
        super().__init__(log)
        self.mon = mon

    def set_params(self, transformer, validation_datagen=None, meta_valid=None):
        super().set_params(transformer)
        self.mon.set_params(transformer, validation_datagen, meta_valid)

    def on_train_begin(self):
        super().on_train_begin()
        self.mon.on_train_begin()

    def on_batch_end(self, metrics=None):
        self.mon.on_batch_end()

    def on_epoch_end(self):
        self.log.append(("validation", self.epoch_id))
        self.mon.on_epoch_end()
        self.epoch_id += 1


class Checkpoint(Callback):
    """ModelCheckpoint with minimize=False (the AP): save_model at epoch 0 and whenever the AP beats the best"""

    def __init__(self, log, path):
        super().__init__(log)
        self.path, self.best, self.saved = path, None, []

    def on_epoch_end(self):
        ap = self.ap()
        self.log.append(("checkpoint", self.epoch_id))
        if self.best is None or ap > self.best or self.epoch_id == 0:
            self.best = ap
            save_model(self.model, self.path)
            self.saved.append(self.epoch_id)
        self.epoch_id += 1


class LRSchedule(Callback):
    """ExponentialLRScheduler with epoch_every=1: a torch ExponentialLR stepped at every epoch end"""

    def __init__(self, log, gamma):
        super().__init__(log)
        self.gamma = gamma

    def set_params(self, transformer, validation_datagen=None, meta_valid=None):
        super().set_params(transformer)
        self.sched = torch.optim.lr_scheduler.ExponentialLR(self.optimizer, self.gamma)

    def on_epoch_end(self):
        self.log.append(("lr", self.epoch_id))
        self.sched.step()
        self.epoch_id += 1


class EarlyStop(Callback):
    """EarlyStopping with minimize=False: break once the AP has not beaten the best for more than `patience` epochs"""

    def __init__(self, log, patience):
        super().__init__(log)
        self.patience, self.best, self.since, self.stop = patience, None, 0, False

    def on_epoch_end(self):
        ap = self.ap()
        self.log.append(("early stopping", self.epoch_id))
        if self.best is None or ap > self.best:
            self.best, self.since = ap, 0
        else:
            self.since += 1
        self.stop = self.since > self.patience
        self.epoch_id += 1

    def training_break(self):
        return self.stop


class CallbackList:
    def __init__(self, callbacks):
        self.callbacks = callbacks

    def __getattr__(self, name):
        def call(*args, **kwargs):
            out = [getattr(c, name)(*args, **kwargs) for c in self.callbacks]
            return any(out) if name == "training_break" else None
        return call


def ap_rules(aps, patience):
    """the stand-ins' rules on a list of epoch APs -> (epochs whose end saves a checkpoint, epochs run): a checkpoint at
    epoch 0 and at every AP above the best; a stop once more than `patience` epochs in a row did not beat the best"""
    best, saved, since = None, [], 0
    for e, ap in enumerate(aps):
        if best is None or ap > best:
            best, since = ap, 0
            saved.append(e)
        else:
            since += 1
        if since > patience:
            return saved, e + 1
    return saved, len(aps)


def assert_released(cuda, before, what):
    """nothing of a ResNet101 model is left on the device: at most 256 MiB more allocated than `before`"""
    free_device_memory()
    left = torch.cuda.memory_allocated(cuda) - before
    assert left < 2 ** 28, "%.2f GiB more allocated after %s than before it" % (left / 2 ** 30, what)


def test_fit_equals_a_hand_driven_loop(mcb, cuda, tmp_path, monkeypatch):
    """The hand-driven loop runs first: it trains RAN epochs, sets the lr each epoch and makes save_model's round trip
    after epochs 0 and 1.  A separately built eval plan gives each epoch's validation logits; the ground truth is every
    other detection of epoch 1, and the oracle chain gives every epoch's AP.  By the stand-ins' rules those APs must
    save checkpoints after epochs 0 and 1 and stop fit() after epoch RAN - 1 of EPOCHS.  fit() then runs with the
    stand-ins, and must give the same losses, epoch-end states, APs, checkpoints and stop, with epoch 1's state on
    disk: a checkpoint written mid-run, after steps of both captured shapes and one earlier round trip."""
    import pandas as pd
    import bench
    from mcb200.models import PyTorchUNetWeighted
    EPOCHS, RAN, STEPS, GAMMA, PATIENCE, SAVES = 4, 3, 2, 0.9, 0, [0, 1]
    sd = seeded_sd(ENCODER)
    epochs = [train_batches(SEED + 100 + 10 * e) for e in range(EPOCHS)]
    extra = batch(SEED + 99, N_TRAIN)
    assert [len(b[0]) for b in epochs[0]] == [20, 20, 7]
    cfg = bench.unet_config(ENCODER)
    cfg["training_config"] = {"epochs": EPOCHS}
    free_device_memory()
    before = torch.cuda.memory_allocated(cuda)

    # the hand-driven loop: the same batches, the lr set each epoch, save_model after epochs 0 and 1
    model = PyTorchUNetWeighted(**cfg)
    model.model.load_state_dict(sd)
    model._to_device()
    net = model.model = nn.DataParallel(model.model, device_ids=[cuda.index or 0])
    layout = arena_layout(model._net())
    group = model.optimizer.param_groups[0]
    hand_path = str(tmp_path / "hand.torch")
    losses, hand, states = [], [], []
    for e in range(RAN):
        for X, T in epochs[e]:
            losses.append(host(model._fit_loop([X, T])["sum"]))
        hand.append(state_of(model, losses[-1]))
        states.append(host_state(net))
        if e in SAVES:
            save_model(net, hand_path)
        group["lr"] *= GAMMA
    hand_lr = group["lr"]
    del model, net, group
    assert_released(cuda, before, "the hand-driven loop")

    # each epoch's validation through a separate eval plan and the oracle chain; the ground truth from epoch 1
    ev = EvalPlan()
    results = [oracle_results(ev.logits(st, cuda), monkeypatch) for st in states]
    del ev
    assert_released(cuda, before, "the eval plan")
    data_dir = str(tmp_path)
    gt = write_ground_truth(results[1], data_dir)
    want = [oracle_ap(gt, r) if r else 0.0 for r in results]
    expect_saved, expect_ran = ap_rules(want, PATIENCE)
    print("detections per epoch %s, oracle APs %s" % ([len(r) for r in results], want))
    assert (expect_saved, expect_ran) == (SAVES, RAN), "the ground truth must make epoch 1 the best and stop fit() " \
        "after epoch %d: checkpoints %s, %d epochs" % (RAN - 1, expect_saved, expect_ran)

    # fit() with the stand-ins, in the order of the reference's callbacks_unet
    path = str(tmp_path / "checkpoints" / "unet.torch")
    os.makedirs(os.path.dirname(path))
    log = []
    snaps, ckpt = Snapshots(log), Checkpoint(log, path)
    cbs = CallbackList([snaps, Validation(log, monitor(data_dir)), ckpt, LRSchedule(log, GAMMA), EarlyStop(log, PATIENCE)])
    model = PyTorchUNetWeighted(**cfg, callbacks=cbs)
    model.model.load_state_dict(sd)
    loader = Loader(epochs, extra)
    model.fit((loader, STEPS), validation_datagen=(val_batches(), None),
              meta_valid=pd.DataFrame({"ImageId": IMAGE_IDS}))
    aps = [model.validation_loss[e]["sum"] for e in sorted(model.validation_loss)]
    fit_lr = model.optimizer.param_groups[0]["lr"]
    fit_losses, fit_states, saved = snaps.losses, snaps.epochs, ckpt.saved
    del model, cbs, snaps, ckpt          # the callbacks hold the transformer, its model and its optimizer
    assert_released(cuda, before, "fit()")
    print("fit(): APs %s, checkpoints after epochs %s, %d epochs run" % ([float(a[0]) for a in aps], saved,
                                                                       len(fit_states)))

    assert [a.item() for a in aps] == [torch.tensor([w], dtype=torch.float32).item() for w in want]
    assert saved == SAVES and len(fit_states) == RAN, (saved, len(fit_states))
    assert loader.drawn == [(e, i) for e in range(RAN) for i in range(STEPS + 1)], loader.drawn
    order = ["snapshot", "validation", "checkpoint", "lr", "early stopping"]
    assert log == [(name, e) for e in range(RAN) for name in order], log
    assert fit_lr == hand_lr
    assert len(losses) == len(fit_losses) == 3 * RAN
    for i, (a, b) in enumerate(zip(fit_losses, losses)):
        assert same_bits(a, b), "batch %d: fit loss %r, hand-driven %r" % (i + 1, a, b)
    compare_runs(layout, hand, fit_states, "fit() against the hand-driven loop, epoch end")
    bad = state_mismatches(states[SAVES[-1]], torch.load(path, map_location="cpu"))
    assert not bad, "the checkpoint on disk is not epoch %d's state: %s" % (SAVES[-1], bad[:10])
