"""Mirror of the reference's model transformers (src/models.py:50-209 over
src/steps/pytorch/models.py:16-171) and losses (src/models.py:310-454,
src/steps/pytorch/validation.py:8-28) on the H100 path.

Same constructor (architecture_config, training_config, callbacks_config), same fit / transform / load / save /
_fit_loop / _transform surface and attributes (.model, .optimizer, .loss_function, .output_names, .callbacks), so
src/pipelines.py builds `Step(name='unet', transformer=PyTorchUNet(**config.unet), ...)` unchanged.

The train step (`_fit_loop`) is one fused device sequence: forward plan -> two-phase loss kernels -> backward plan ->
fused Adam, replayed from CUDA graphs; under torch.distributed (one process per GPU) the Dice sums and the gradient
arena are all-reduced over NCCL.  Nothing here computes on the CPU."""
import math
import os
import shutil
import warnings
from functools import partial

import numpy as np
import torch
import torch.distributed as dist
from torch import nn, optim

from . import _lib as L
from . import ops
from .unet_models import AlbuNet, UNetResNet

# registry of src/models.py:22-47, AlbuNet and ResNet entries (pretrained weights need a network: load a checkpoint
# instead)
PRETRAINED_NETWORKS = {
    'AlbuNet': {'model': AlbuNet,
                'model_config': {'num_classes': 2, 'pretrained': False, 'is_deconv': True},
                'init_weights': False},
    'ResNet34': {'model': UNetResNet,
                 'model_config': {'encoder_depth': 34, 'num_classes': 2, 'num_filters': 32, 'dropout_2d': 0.0,
                                  'pretrained': False, 'is_deconv': True, },
                 'init_weights': False},
    'ResNet101': {'model': UNetResNet,
                  'model_config': {'encoder_depth': 101, 'num_classes': 2, 'num_filters': 32, 'dropout_2d': 0.0,
                                   'pretrained': False, 'is_deconv': True, },
                  'init_weights': False},
    'ResNet152': {'model': UNetResNet,
                  'model_config': {'encoder_depth': 152, 'num_classes': 2, 'num_filters': 32, 'dropout_2d': 0.0,
                                   'pretrained': False, 'is_deconv': True, },
                  'init_weights': False},
}


# ---------------------------------------------------------------------------------------------------------------------
# losses (autograd-compatible wrappers over the two-phase CUDA kernels)
# ---------------------------------------------------------------------------------------------------------------------
class _FusedLoss(torch.autograd.Function):
    """loss of the LOCAL batch (what the reference's validation callbacks expect from `loss_function(outputs, target)`,
    src/steps/pytorch/validation.py:47-80, possibly on one rank only); the cross-rank Dice / CE sums of multi-GPU
    training are all-reduced by FusedTrainStep, never here (pass sync=True in cfg to opt in)."""

    @staticmethod
    def forward(ctx, logits, target, mode, cfg):
        logits = logits.contiguous().float()
        target = target.contiguous().float()
        sums = torch.zeros(4, dtype=torch.float64, device=logits.device)
        ops.loss_partials(logits, target, sums, mode=mode, **cfg)
        world = 1
        if cfg.get("sync", False) and dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
            dist.all_reduce(sums)
            world = dist.get_world_size()
        dlogits = torch.empty_like(logits)
        loss = torch.empty((), dtype=torch.float32, device=logits.device)
        n, _, h, w = logits.shape
        ops.loss_grad(logits, target, sums, dlogits, loss, global_pixels=n * h * w * world, mode=mode, **cfg)
        ctx.save_for_backward(dlogits)
        return loss

    @staticmethod
    def backward(ctx, g):
        (dlogits,) = ctx.saved_tensors
        return dlogits * g, None, None, None


def _size_c(imsize):
    return math.sqrt(imsize[0] * imsize[1]) / 2.0


def multiclass_segmentation_loss(output, target):
    """src/steps/pytorch/validation.py:25-28 — plain 2-class cross entropy; target (N,1,H,W)"""
    return _FusedLoss.apply(output, target, 1, {})


def mixed_dice_cross_entropy_loss(output, target, dice_weight=0.5, dice_loss=None, cross_entropy_weight=0.5,
                                  cross_entropy_loss=None, smooth=0, dice_activation='softmax', w0=50.0, sigma=10.0,
                                  imsize=(256, 256)):
    """src/models.py:384-418 in the configuration PyTorchUNetWeighted builds (src/models.py:149-161): Dice on class 1
    (of the softmax, or of the sigmoid of the class-1 logit) + distance/size-weighted cross entropy; target (N,3,H,W) =
    [mask, distances, sizes]"""
    ops.dice_activation_code(dice_activation)
    cfg = dict(w0=w0, sigma=sigma, size_c=_size_c(imsize), dice_weight=dice_weight, ce_weight=cross_entropy_weight,
               dice_smooth=smooth, dice_activation=dice_activation)
    return _FusedLoss.apply(output, target, 0, cfg)


# ---------------------------------------------------------------------------------------------------------------------
# minimal callback plumbing (the reference's CallbackList is host-side bookkeeping and plugs in unchanged)
# ---------------------------------------------------------------------------------------------------------------------
class NullCallbacks:
    def set_params(self, transformer, validation_datagen=None, meta_valid=None):
        self.transformer = transformer

    def on_train_begin(self, *a, **k): pass
    def on_train_end(self, *a, **k): pass
    def on_epoch_begin(self, *a, **k): pass
    def on_epoch_end(self, *a, **k): pass
    def on_batch_begin(self, *a, **k): pass
    def on_batch_end(self, *a, **k): pass
    def training_break(self, *a, **k): return False


def callbacks_unet(callbacks_config):
    """src/models.py:295-307: the reference builds its CallbackList (timing, training / validation monitors, checkpoint,
    exponential LR schedule, early stopping, neptune) from `callbacks_config` in the transformer's constructor
    (src/models.py:60).  Those callbacks are host-side bookkeeping of the reference package and plug in unchanged, so
    they are taken from it when it is importable (i.e. whenever this transformer runs inside the reference's pipeline);
    outside the reference tree there is nothing to build them from, which is said loudly, not silently."""
    if not callbacks_config:
        return NullCallbacks()
    try:
        from src.models import callbacks_unet as reference_callbacks_unet
    except Exception as e:  # reference package (or one of its dependencies) not importable
        warnings.warn("mcb200: callbacks_config given but the reference package `src` is not importable (%s: %s); "
                      "training runs WITHOUT checkpointing / validation / LR schedule / early stopping. Pass "
                      "`callbacks=` explicitly or run inside the reference tree." % (type(e).__name__, e),
                      RuntimeWarning, stacklevel=3)
        return NullCallbacks()
    return reference_callbacks_unet(callbacks_config)


def release_captured_graphs(transformer):
    """drop every captured CUDA graph / launch plan of a transformer.  Call it before
    torch.distributed.destroy_process_group(): graphs that captured NCCL collectives keep the communicator busy and the
    teardown waits on them forever."""
    import gc
    transformer._fused = None
    transformer._fused_cache = {}
    net = transformer._net()
    net._plans = {}
    gc.collect()
    if torch.cuda.is_available():
        torch.cuda.synchronize()


def weight_regularization_unet(model, regularize, weight_decay_conv2d):
    """src/models.py:287-292"""
    if regularize:
        return [{'params': model.parameters(), 'weight_decay': weight_decay_conv2d}]
    return [model.parameters()]


class Model:
    """src/steps/pytorch/models.py:16-171 (Model) on the H100 path"""

    def __init__(self, architecture_config, training_config, callbacks_config):
        self.architecture_config = architecture_config
        self.training_config = training_config
        self.callbacks_config = callbacks_config
        self.model = None
        self.optimizer = None
        self.loss_function = None
        self.callbacks = None
        self.validation_loss = {}
        self._fused = None          # the FusedTrainStep of the most recent batch shape
        self._fused_cache = {}      # (X.shape, target.shape) -> FusedTrainStep (the last batch of an epoch is smaller)
        self._opt_state = None      # Adam moments + step count, arena-sized, shared by every cached step
        self._step = 0

    @property
    def output_names(self):
        return [name for (name, func, weight) in self.loss_function]

    # ---- BaseTransformer surface (src/steps/base.py:254-269)
    def fit_transform(self, *args, **kwargs):
        self.fit(*args, **kwargs)
        return self.transform(*args, **kwargs)

    def _initialize_model_weights(self):
        return None  # pretrained-encoder configs replace the initialiser by a no-op (src/models.py:101)

    def _net(self):
        return self.model.module if isinstance(self.model, nn.DataParallel) else self.model

    def fit(self, datagen, validation_datagen=None, meta_valid=None):
        self._initialize_model_weights()
        self._to_device()
        if not isinstance(self.model, nn.DataParallel):
            # src/models.py:65: the reference wraps the net, so callbacks see `transformer.model` as a DataParallel and
            # ModelCheckpoint writes `module.`-prefixed keys.  One process drives one GPU here: the wrapper has a single
            # device and forwards straight to the module.
            dev = self._net()._p32.device
            self.model = nn.DataParallel(self.model, device_ids=[dev.index if dev.index is not None else 0])
        self.callbacks.set_params(self, validation_datagen=validation_datagen, meta_valid=meta_valid)
        self.callbacks.on_train_begin()
        batch_gen, steps = datagen
        for epoch_id in range(self.training_config['epochs']):
            self.callbacks.on_epoch_begin()
            for batch_id, data in enumerate(batch_gen):
                self.callbacks.on_batch_begin()
                metrics = self._fit_loop(data)
                self.callbacks.on_batch_end(metrics=metrics)
                if batch_id == steps:
                    break
            self.callbacks.on_epoch_end()
            if self.callbacks.training_break():
                break
        self.callbacks.on_train_end()
        return self

    def _to_device(self):
        if not torch.cuda.is_available():
            raise RuntimeError("the H100 path needs a CUDA device; there is no CPU fallback")
        net = self._net()
        if not net._p32.is_cuda:
            params_before = [p for _, p, _ in net._arena_params()]
            net.cuda()
            # parameters keep their identity (only .data moved), so the optimizer's references stay valid
            assert all(a is b for a, b in zip(params_before, [p for _, p, _ in net._arena_params()]))

    # ---- fused train step
    def _loss_spec(self):
        """(mode, cfg) when the configured loss is one the fused kernels implement, else None"""
        return getattr(self, "_fused_loss", None)

    def _fit_loop(self, data):
        """src/steps/pytorch/models.py:76-113: H2D, zero_grad, forward, loss, backward, optimizer.step"""
        X = data[0]
        targets = data[1:]
        self._to_device()
        net = self._net()
        net.train()
        dev = net._p32.device
        target = targets[0]
        spec = self._loss_spec()
        if spec is None:
            X = X.to(dev, non_blocking=True).float()
            target = target.to(dev, non_blocking=True).float()
            # arbitrary user loss: CUDA forward/backward through the autograd bridge + the torch optimizer
            self.optimizer.zero_grad()
            out = net(X)
            (name, loss_function, weight) = self.loss_function[0]
            batch_loss = loss_function(out, target) * weight
            batch_loss.backward()
            self.optimizer.step()
            return {'sum': batch_loss.detach().reshape(1)}   # shape (1,), like the fused path (callbacks index [0])
        self._fused = self._fused_step(net, X.shape, target.shape, spec)
        group = self.optimizer.param_groups[0]
        loss = self._fused.step(X, target, lr=group['lr'], betas=group.get('betas', (0.9, 0.999)),
                                eps=group.get('eps', 1e-8), weight_decay=group.get('weight_decay', 0.0))
        return {'sum': loss}

    def _fused_step(self, net, x_shape, t_shape, spec):
        """the captured train step for this batch shape.  Adam's moments and step count live on the transformer, not in
        the captured step: a partial last batch (the reference's DataLoader has no drop_last, src/loaders.py:220) or a
        device round trip of the model (ModelCheckpoint -> save_model: model.cpu(); save; model.cuda()) re-captures
        graphs but never resets the optimizer."""
        gen = net._generation
        st = self._opt_state
        if st is None:
            st = self._opt_state = AdamState(net)
        elif st.generation != gen or st.m.device != net._p32.device or st.m.numel() != net._p32.numel():
            st.rebind(net)              # arenas were re-created: carry m / v / t over, drop steps that baked pointers in
            self._fused_cache = {}
        key = (tuple(x_shape), tuple(t_shape))
        fused = self._fused_cache.get(key)
        if fused is None:
            fused = self._fused_cache[key] = FusedTrainStep(net, x_shape, t_shape, spec[0], spec[1], st)
        return fused

    # ---- inference (src/steps/pytorch/models.py:115-142)
    def _transform(self, datagen, validation_datagen=None):
        self._to_device()
        net = self._net()
        net.eval()
        batch_gen, steps = datagen
        outputs = {}
        for batch_id, data in enumerate(batch_gen):
            X = data[0] if isinstance(data, (list, tuple)) else data
            with torch.no_grad():
                out = net(X.to(net._p32.device).float())
            outputs.setdefault(self.output_names[0], []).append(out)
            if batch_id == steps:
                break
        net.train()
        return {'{}_prediction'.format(name): torch.cat(outs, 0) for name, outs in outputs.items()}

    def load(self, filepath):
        """src/steps/pytorch/models.py:148-160 — accepts checkpoints saved from the DataParallel wrapper
        (`module.`-prefixed keys, src/steps/pytorch/utils.py:67-75) as well as plain ones"""
        net = self._net()
        net.eval()
        sd = torch.load(filepath, map_location='cpu')
        sd = {(k[7:] if k.startswith('module.') else k): v for k, v in sd.items()}
        net.load_state_dict(sd)
        if torch.cuda.is_available():
            self._to_device()
            net.refresh_operands()   # the captured steps read the bf16 operand copy, which only Adam refreshes
        return self

    def save(self, filepath):
        """src/steps/pytorch/models.py:162-171 + save_model: state_dict with the `module.` prefix the reference's
        DataParallel checkpoints carry"""
        checkpoint_callback = (self.callbacks_config or {}).get('model_checkpoint')
        if checkpoint_callback and os.path.exists(checkpoint_callback.get('filepath', '')):
            shutil.copyfile(checkpoint_callback['filepath'], filepath)
            return
        sd = {'module.' + k: v.cpu() for k, v in self._net().state_dict().items()}
        os.makedirs(os.path.dirname(os.path.abspath(filepath)), exist_ok=True)
        torch.save(sd, filepath)


class BasePyTorchUNet(Model):
    """src/models.py:50-101"""

    def __init__(self, architecture_config, training_config, callbacks_config, callbacks=None):
        super().__init__(architecture_config, training_config, callbacks_config)
        self.set_model()
        self.weight_regularization = weight_regularization_unet
        self.optimizer = optim.Adam(self.weight_regularization(self.model, **architecture_config['regularizer_params']),
                                    **architecture_config['optimizer_params'])
        self.loss_function = None
        self.callbacks = callbacks if callbacks is not None else callbacks_unet(self.callbacks_config)

    def transform(self, datagen, validation_datagen=None, *args, **kwargs):
        """src/models.py:88-92: logits -> softmax probabilities, as numpy like the reference"""
        outputs = self._transform(datagen, validation_datagen)
        return {name: ops.softmax2(pred.contiguous()).cpu().numpy() for name, pred in outputs.items()}

    def set_model(self):
        encoder = self.architecture_config['model_params']['encoder']
        if encoder not in PRETRAINED_NETWORKS:
            raise NotImplementedError("the registry holds the AlbuNet and ResNet34/101/152 encoders; the VGG11 and VGG16 "
                                      "U-Nets are not registered (build mcb200.unet_models.UNet11 / UNetVGG16 and "
                                      "drive them with FusedTrainStep) (got %r)" % (encoder,))
        config = PRETRAINED_NETWORKS[encoder]
        self.model = config['model'](**config['model_config'])
        self._initialize_model_weights = lambda: None


class PyTorchUNet(BasePyTorchUNet):
    """src/models.py:104-107"""

    def __init__(self, architecture_config, training_config, callbacks_config, callbacks=None):
        super().__init__(architecture_config, training_config, callbacks_config, callbacks)
        self.loss_function = [('multichannel_map', multiclass_segmentation_loss, 1.0)]
        self._fused_loss = (1, {})


class PyTorchUNetWeighted(BasePyTorchUNet):
    """src/models.py:149-161"""

    def __init__(self, architecture_config, training_config, callbacks_config, callbacks=None):
        dice = architecture_config['dice']
        activation = dice.get('dice_activation', 'softmax')
        # checked here, not at the first loss call as in the reference: the fused train step and the autograd loss must
        # both compute the configured Dice, so no step may run on a config neither implements
        ops.dice_activation_code(activation)
        super().__init__(architecture_config, training_config, callbacks_config, callbacks)
        wce = architecture_config['weighted_cross_entropy']
        lw = architecture_config['loss_weights']
        loss = partial(mixed_dice_cross_entropy_loss, dice_weight=lw['dice_mask'], cross_entropy_weight=lw['bce_mask'],
                       smooth=dice['smooth'], dice_activation=activation, w0=wce['w0'], sigma=wce['sigma'],
                       imsize=tuple(wce['imsize']))
        self.loss_function = [('multichannel_map', loss, 1.0)]
        self._fused_loss = (0, dict(w0=float(wce['w0']), sigma=float(wce['sigma']), size_c=_size_c(wce['imsize']),
                                    dice_weight=float(lw['dice_mask']), ce_weight=float(lw['bce_mask']),
                                    dice_smooth=float(dice['smooth']), dice_activation=activation))


class _StreamMixin:
    """generator-returning inference of src/models.py:110-146,164-209"""

    def transform(self, datagen, validation_datagen=None, *args, **kwargs):
        if len(self.output_names) != 1:
            raise NotImplementedError
        return {'{}_prediction'.format(self.output_names[0]): self._stream(datagen)}

    def _stream(self, datagen):
        self._to_device()
        net = self._net()
        net.eval()
        batch_gen, steps = datagen
        for batch_id, data in enumerate(batch_gen):
            X = data[0] if isinstance(data, (list, tuple)) else data
            with torch.no_grad():
                out = net(X.to(net._p32.device).float())
            probs = ops.softmax2(out.contiguous()).cpu().numpy()
            for p in probs:
                yield p
            if batch_id == steps:
                break
        net.train()


class PyTorchUNetStream(_StreamMixin, PyTorchUNet):
    pass


class PyTorchUNetWeightedStream(_StreamMixin, PyTorchUNetWeighted):
    pass


# ---------------------------------------------------------------------------------------------------------------------
# fused train step
# ---------------------------------------------------------------------------------------------------------------------
class AdamState:
    """Adam's first / second moments (fp32, laid out like the master arena) and its step count"""

    def __init__(self, net):
        self.m = torch.zeros_like(net._p32)
        self.v = torch.zeros_like(net._p32)
        self.t = 0
        self.generation = net._generation

    def rebind(self, net):
        if self.m.numel() != net._p32.numel():
            raise RuntimeError("the parameter arena changed size; the optimizer state cannot be carried over")
        self.m = self.m.to(net._p32.device)
        self.v = self.v.to(net._p32.device)
        self.generation = net._generation


class FusedTrainStep:
    """forward plan -> loss partials -> [all-reduce sums] -> loss gradient -> backward plan -> [all-reduce grads] ->
    fused Adam (+ bf16 operand refresh), as CUDA graph segments on the current stream.

    Multi-GPU (torch.distributed initialised, one process per GPU): reference DataParallel semantics are kept for
    BatchNorm (per-replica batch statistics, src/models.py:65) while the loss is global-batch (Dice sums all-reduced,
    CE mean over the global pixel count) and gradients are summed; see DESIGN.md (multi-GPU)."""

    def __init__(self, net, x_shape, t_shape, loss_mode, loss_cfg, opt_state=None):
        self.net = net
        self.opt = opt_state if opt_state is not None else AdamState(net)
        self.key = (tuple(x_shape), tuple(t_shape))
        n, _, h, w = x_shape
        self.plan = net.plan(n, h, w, True)
        dev = net._p32.device
        self.dev = dev
        self.loss_mode, self.loss_cfg = loss_mode, dict(loss_cfg)
        self.target = torch.zeros(t_shape, dtype=torch.float32, device=dev)
        self.sums = torch.zeros(4, dtype=torch.float64, device=dev)
        self.loss = torch.zeros((), dtype=torch.float32, device=dev)
        self.world = dist.get_world_size() if (dist.is_available() and dist.is_initialized()) else 1
        self.graphs = None
        self.pixels = n * h * w
        net.refresh_operands()
        self.launches = None
        self._staging = None
        # single GPU: the Adam update of a finished arena segment (decoder | layer4 | rest) rides on the backward's side
        # stream, inside the graph, overlapping the data-gradient GEMMs of the layers below (HBM-bound next to
        # tensor-bound).  Its step-dependent scalars live in a 3-float device tensor refreshed before every replay.
        # multi-GPU: the all-reduce of a finished arena segment (decoder | layer4 | layer3 | rest) is issued from
        # INSIDE the backward graph, on the side stream behind that segment's weight-gradient GEMMs, and overlaps the
        # data-gradient chain of the layers below.  NCCL-per-BatchNorm SyncBN (MCB_SYNC_BN=1) instead takes a single
        # all-reduce after the backward graph, because its BatchNorm slots are rescaled after the backward pass.
        self.inline_allreduce = self.world > 1 and not (self.plan.sync_bn and not self.plan.sync_nvlink)
        self.adam_in_graph = self.world == 1
        self._hyper = torch.zeros(3, dtype=torch.float32, device=dev)
        # pinned staging ring: a slot is rewritten only after the copy that last read it has executed
        self._hyper_ring = [(torch.zeros(3, dtype=torch.float32).pin_memory(), torch.cuda.Event()) for _ in range(8)]
        self._adam_cfg = None
        self.phase_marks = None

    # segments ----------------------------------------------------------------------------------------------------
    def _seg_forward(self):
        self.plan._run_fwd()

    def _loss_partials(self):
        # outside the graphs: it is the first reader of the target, whose H2D copy overlaps the forward segment
        L.zero(self.sums)
        ops.loss_partials(self.plan.logits, self.target, self.sums, mode=self.loss_mode, **self.loss_cfg)

    def _seg_backward(self):
        ops.loss_grad(self.plan.logits, self.target, self.sums, self.plan.dlogits, self.loss,
                      global_pixels=self.pixels * self.world, mode=self.loss_mode, **self.loss_cfg)
        hooks = None
        if self.adam_in_graph:
            net = self.net
            betas, eps, wd = self._adam_cfg

            def upd(lo, hi):
                return lambda: ops.adam_step_dyn(net._p32[lo:hi], net._g32[lo:hi], self.opt.m[lo:hi], self.opt.v[lo:hi],
                                                 net._w16[lo:hi], self._hyper, betas, eps, wd, 1.0)
            hooks = {last: upd(lo, hi) for _, last, lo, hi in self.plan.bwd_segments()}
        works = []
        if self.inline_allreduce:
            # the all-reduce of a finished arena segment is issued from INSIDE the single backward graph, on the side
            # stream behind that segment's weight-gradient GEMMs, and overlaps the data-gradient chain of the layers
            # below; the main stream joins the collectives at the end of the graph.  (Multi-GPU runs have not been
            # measured on the H100.)
            g32 = self.net._g32
            hooks = {last: (lambda lo=lo, hi=hi: works.append(dist.all_reduce(g32[lo:hi], async_op=True)))
                     for _, last, lo, hi in self.plan.bwd_segments()}
        self.plan._run_bwd(hooks=hooks)
        for wk in works:
            wk.wait()

    def _adam(self, lr, betas, eps, weight_decay):
        net = self.net
        ops.adam_step(net._p32, net._g32, self.opt.m, self.opt.v, net._w16, self.opt.t, lr, betas, eps, weight_decay, 1.0)

    def _capture(self):
        gs = []
        from .engine import graph_capture
        for seg in (self._seg_forward, self._seg_backward):
            g = torch.cuda.CUDAGraph()
            with graph_capture(g, self.dev):      # main chain on a high-priority stream
                seg()
            gs.append(g)
        self.graphs = gs

    def _stage_inputs(self, X, target):
        """host batches go through a copy stream into double-buffered staging tensors so that the H2D transfer of
        step i+1 overlaps the compute of step i, and the target's transfer overlaps the forward pass of its own step
        (the loss is its first reader); device batches are copied directly.  Returns a callable that makes the target
        visible to the current stream (call it after launching the forward)."""
        cur = torch.cuda.current_stream()
        if X.is_cuda and target.is_cuda:
            self.plan.x_in.copy_(X, non_blocking=True)
            self.target.copy_(target, non_blocking=True)
            return lambda: None
        if self._staging is None:
            self._copy_stream = torch.cuda.Stream(device=self.dev)
            self._staging = [(torch.empty_like(self.plan.x_in), torch.empty_like(self.target),
                              torch.cuda.Event(), torch.cuda.Event(), torch.cuda.Event()) for _ in range(2)]
            self._stage_i = 0
        sx, st, ev_x, ev_t, ev_consumed = self._staging[self._stage_i]
        self._stage_i ^= 1
        cs = self._copy_stream
        cs.wait_event(ev_consumed)  # the compute stream finished reading this slot (no-op before first use)
        with torch.cuda.stream(cs):
            sx.copy_(X.float() if X.dtype != torch.float32 else X, non_blocking=True)
            ev_x.record(cs)
            st.copy_(target.float() if target.dtype != torch.float32 else target, non_blocking=True)
            ev_t.record(cs)
        cur.wait_event(ev_x)
        self.plan.x_in.copy_(sx, non_blocking=True)

        def finish_target():
            cur.wait_event(ev_t)
            self.target.copy_(st, non_blocking=True)
            ev_consumed.record(cur)
        return finish_target

    def step(self, X, target, lr, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0):
        if self.adam_in_graph:
            cfg = (tuple(betas), eps, weight_decay)
            if self._adam_cfg is None:
                self._adam_cfg = cfg
            elif self._adam_cfg != cfg:   # baked into the captured launches; refused before the step counts
                raise RuntimeError("Adam betas / eps / weight_decay changed after the train step was captured")
        finish_target = self._stage_inputs(X, target)
        self.opt.t += 1
        t = self.opt.t
        if self.adam_in_graph:
            host, ev = self._hyper_ring[t % len(self._hyper_ring)]
            ev.synchronize()
            host[0], host[1], host[2] = ops.adam_hyper(lr, betas, t)
            self._hyper.copy_(host, non_blocking=True)
            ev.record()
        first = self.graphs is None
        marks = self.phase_marks            # bench.py: CUDA events at the phase boundaries of a step (None = off)

        def mark(name):
            if marks is not None:
                e = torch.cuda.Event(enable_timing=True)
                e.record()
                marks.append((name, e))
        mark("start")
        if first:
            self._seg_forward()
        else:
            self.graphs[0].replay()
        mark("forward")
        finish_target()
        self._loss_partials()
        if self.world > 1:
            dist.all_reduce(self.sums)
        mark("loss sums")
        if first:
            self._seg_backward()
        else:
            self.graphs[1].replay()
        if self.world > 1 and not self.inline_allreduce:
            if self.plan.sync_bn and not self.plan.sync_nvlink:
                # the BatchNorm slots already hold GLOBAL sums (engine.Plan.sync_bn_grads): pre-divide so that the
                # arena-wide SUM below leaves them unchanged
                torch._foreach_mul_(self.plan.bn_grad_slices(), 1.0 / self.world)
            dist.all_reduce(self.net._g32)   # gradients of the global-batch loss = sum of the per-rank contributions
        mark("backward (+ in-graph Adam / all-reduce)")
        if not self.adam_in_graph:
            self._adam(lr, betas, eps, weight_decay)
            mark("adam")
        if first:
            torch.cuda.synchronize()
            self._capture()
        # shape (1,): the reference's callbacks read `loss.data.cpu().numpy()[0]` (src/steps/pytorch/callbacks.py:134)
        return self.loss.reshape(1).clone()

    def count_launches(self):
        """kernel launches of one step (our kernels + memsets issued by the plan)"""
        return self.plan.launches_fwd + self.plan.launches_bwd + (6 if self.adam_in_graph else 4)
