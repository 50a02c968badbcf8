"""CPU test of the launch plans' complete launch trace (mcb200.engine.Plan): every entry point the forward and the
backward call, with every argument, on the stream it is issued on, and every event record and wait between the streams.

The plan allocates its tensors on the net's device, so a CPU net builds one without a GPU.  The library calls, the CUDA
streams and events and (for SyncBN) torch.distributed are replaced by recorders; pointers are recorded as (allocation
ordinal in order of first appearance, byte offset) over the allocations the plan may legitimately address, so the trace
is independent of where the allocator put them.  A change of a buffer, a flag, a shape, a stream placement or an event
edge changes the trace's sha256."""
import bisect
import ctypes as C
import hashlib
import json
import types

import pytest
import torch
from torch import nn

_BYREF = type(C.byref(C.c_int()))    # a struct passed by reference (ops.bn_train_apply)


class _Stream:
    def __init__(self, name):
        self.name = name

    def wait_event(self, ev):
        _REC.log.append(("wait", self.name, ev.idx))


class _Event:
    def __init__(self, *args, **kwargs):
        self.idx = _REC.n_events
        _REC.n_events += 1

    def record(self, stream=None):
        _REC.log.append(("record", self.idx, (stream or _REC.cur).name))


class _StreamCtx:
    def __init__(self, s):
        self.s = s

    def __enter__(self):
        self.prev, _REC.cur = _REC.cur, self.s

    def __exit__(self, *exc):
        _REC.cur = self.prev


class _Recorder:
    def __init__(self, net, plan):
        tensors = [net._p32, net._g32, net._w16, plan._stats_arena, plan.x_in, plan.logits, plan.dlogits]
        tensors += [b for m in net.modules() if isinstance(m, nn.BatchNorm2d) for b in (m.running_mean, m.running_var)]
        tensors += [t for t in plan._keep if isinstance(t, torch.Tensor)]
        spans = {}
        for t in tensors:
            st = t.untyped_storage()
            if st.nbytes():
                spans[st.data_ptr()] = st.nbytes()
        self.bases = sorted(spans)
        self.sizes = [spans[b] for b in self.bases]
        self.ordinal = {}
        self.log = []
        self.n_events = 0
        self.n_streams = 0
        self.cur = _Stream("main")

    def ptr(self, p):
        if p is None or p == 0:
            return None
        i = bisect.bisect_right(self.bases, p) - 1
        assert i >= 0 and p < self.bases[i] + self.sizes[i], "pointer %#x lies in no allocation of the plan" % p
        base = self.bases[i]
        return [self.ordinal.setdefault(base, len(self.ordinal)), p - base]

    def tensor(self, t):
        return [self.ptr(t.data_ptr()), t.numel(), str(t.dtype)]

    def struct(self, s):
        out = []
        for name, ty in s._fields_:
            v = getattr(s, name)
            if ty is C.c_void_p:
                v = self.ptr(v)
            elif issubclass(ty, C.Array):
                v = [self.ptr(x) for x in v] if ty._type_ is C.c_void_p else list(v)
            out.append([name, v])
        return out

    def bn_table(self, p, n):
        rows = list((C.c_longlong * (7 * n)).from_address(p))
        return [[self.ptr(x) for x in rows[7 * i:7 * i + 6]] + [rows[7 * i + 6]] for i in range(n)]

    # replacements of mcb200._lib.call / fcall / zero
    def call(self, name, args=None, *extra):
        self.log.append(("call", self.cur.name, name, self.struct(args) if args is not None else None, list(extra)))

    def fcall(self, name, *args):
        from mcb200 import _lib as L
        types_ = getattr(L.lib, name).argtypes
        if name == "mcb_bn_eval_params_batched":
            rec = [self.bn_table(args[0], args[1])] + list(args[1:])
        else:
            rec = []
            for ty, v in zip(types_, args):
                if isinstance(v, _BYREF):
                    rec.append(self.struct(v._obj))
                elif ty is C.c_void_p:
                    rec.append(self.ptr(v))
                else:
                    rec.append(v)
        self.log.append(("fcall", self.cur.name, name, rec))

    def zero(self, t):
        self.log.append(("zero", self.cur.name, self.tensor(t)))

    def new_stream(self, *args, **kwargs):
        self.n_streams += 1
        return _Stream("side%d" % self.n_streams)


_REC = None


def _trace(monkeypatch, net, n, h, w, training, world=1):
    """the launch trace of one forward and (training) one backward with FusedTrainStep's hooks"""
    global _REC
    from mcb200 import _lib as L
    from mcb200 import engine, ops
    if world > 1:
        monkeypatch.setenv("MCB_SYNC_BN", "1")
        monkeypatch.setattr(engine, "dist", types.SimpleNamespace(
            is_available=lambda: True, is_initialized=lambda: True, get_world_size=lambda: world,
            all_reduce=lambda t, *a, **k: _REC.log.append(("all_reduce", _REC.cur.name, _REC.tensor(t)))))

    def chk(t, dtype=torch.bfloat16):
        assert t.is_contiguous() and t.dtype == dtype, (t.is_contiguous(), t.dtype)
        return t
    monkeypatch.setattr(ops, "_chk", chk)
    plan = net.plan(n, h, w, training)
    assert plan.sync_bn == (world > 1)
    _REC = rec = _Recorder(net, plan)
    monkeypatch.setattr(L, "call", rec.call)
    monkeypatch.setattr(L, "fcall", rec.fcall)
    monkeypatch.setattr(L, "zero", rec.zero)
    monkeypatch.setattr(torch.cuda, "current_stream", lambda *a, **k: _REC.cur)
    monkeypatch.setattr(torch.cuda, "Stream", rec.new_stream)
    monkeypatch.setattr(torch.cuda, "Event", _Event)
    monkeypatch.setattr(torch.cuda, "stream", _StreamCtx)
    plan._run_fwd()
    if training:
        rec.log.append(("backward",))
        hooks = {last: (lambda lo=lo, hi=hi: _REC.log.append(("hook", _REC.cur.name, lo, hi)))
                 for _, last, lo, hi in plan.bwd_segments()}
        plan._run_bwd(hooks)
    _REC = None
    return rec.log


def _digest(log):
    return hashlib.sha256(json.dumps(log).encode()).hexdigest()


def _net(arch):
    from mcb200.unet_models import AlbuNet, UNet11, UNetResNet, UNetVGG16
    with torch.random.fork_rng():
        torch.manual_seed(0)
        if arch.startswith("resnet"):
            return UNetResNet(int(arch[6:]), 2, 32, 0.0, False, True)
        if arch == "albunet":
            return AlbuNet(num_classes=2, pretrained=False, is_deconv=True)
        if arch == "vgg11":
            return UNet11(num_classes=2, pretrained=False)
        return UNetVGG16(num_classes=2, dropout_2d=0.0, pretrained=False, is_deconv=True)


SIZE = {"resnet34": 320, "resnet101": 320, "resnet152": 320, "albunet": 256, "vgg11": 256, "vgg16": 256}

# sha256 of the launch trace of every plan at batch 2, as the planner built it before it was split into a core and one
# builder per encoder family
TRACE_SHA256 = {
    "resnet34-train": "eb900e166a08592c336757306ba369f68a47bc37350ad506d24801b841a036a2",
    "resnet34-eval": "31601e826ff6d98b81cad9a384b51c0b66f4bb27258198764a58151e90ea9cb2",
    "resnet101-train": "323d7dcd7b6e5639767b7adf0308788ea375b7a1ab7c040c740ee65f22e1cba0",
    "resnet101-eval": "8a34b4b86e9644e7323a840f4ac1d337726abbca8a5dfe522c1c556df67cbe08",
    "resnet152-train": "110c4fbf2a8d4537cf9c9a1f960b7c8a40feeb0831f1e8bde176198e6e0f7114",
    "resnet152-eval": "0ae7340220d80ea67ee3a97a533bcf466333a94f371712ebeb45b1060dcf46b6",
    "albunet-train": "7feb2abd65be323dc00815cecada649d1f07b1288b773395d9f16f872e838494",
    "albunet-eval": "edba386908334eacffc85abc4a01fd52be34e5f472a03202faf16e15d22c660d",
    "vgg11-train": "134432dc62c45ae16bedc76031de2978b5676989655c24249d51a765022767c6",
    "vgg11-eval": "627ba3cbb73b3df8f41150e462e7d30bd286770e077f9ab44f53eaf5e01782e9",
    "vgg16-train": "cab0a05aa625a6bc9d00595e35b51a9ca4d78759c7d4d0ca3940e2efa5691869",
    "vgg16-eval": "4c01cd918d92a1171f872d0a6f71d344301a33224a31bafb2d31b5d2f91a9add",
    "resnet34-train-syncbn": "e365c506a3a58a59053cba3bf748b7aa7e4fc240aafa4335722c39cfb00e3e6f",
}


@pytest.mark.parametrize("training", [True, False], ids=["train", "eval"])
@pytest.mark.parametrize("arch", list(SIZE))
def test_launch_trace_is_pinned(mcb, monkeypatch, arch, training):
    log = _trace(monkeypatch, _net(arch), 2, SIZE[arch], SIZE[arch], training)
    key = "%s-%s" % (arch, "train" if training else "eval")
    assert _digest(log) == TRACE_SHA256[key], key


def test_sync_bn_launch_trace_is_pinned(mcb, monkeypatch):
    """MCB_SYNC_BN=1 under a world of 2: one all-reduce of [sum, sum^2] per BatchNorm in the forward, one of
    [dgamma, dbeta] per BatchNorm in the backward"""
    net = _net("resnet34")
    log = _trace(monkeypatch, net, 2, 320, 320, True, world=2)
    n_bn = sum(isinstance(m, nn.BatchNorm2d) for m in net.modules())
    i_bwd = log.index(("backward",))
    assert sum(e[0] == "all_reduce" for e in log[:i_bwd]) == n_bn
    assert sum(e[0] == "all_reduce" for e in log[i_bwd:]) == n_bn
    assert _digest(log) == TRACE_SHA256["resnet34-train-syncbn"]
