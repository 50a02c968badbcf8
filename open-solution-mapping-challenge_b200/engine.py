"""Static launch plans for the U-Nets of unet_models (UNetResNet / AlbuNet through ResNetPlan, and the BatchNorm-free
UNet11 / UNetVGG16 through VGGPlan): every kernel launch of one forward (and its backward) over preallocated
NHWC bf16 buffers, replayable as CUDA graphs.

Data flow per conv+BN unit in training:  z = conv(a_prev) [+ per-channel sum / sumsq in the GEMM epilogue]
-> bn_finalize (batch statistics, running-stat update) -> a = relu(z*scale + shift [+ residual]) in one pass.
Backward mirrors torch autograd of src/unet_models.py:385-403: per unit a reduction
(dbeta, dgamma with the ReLU mask folded in), one elementwise pass producing dz, then the wgmma dgrad and
split-K wgrad GEMMs; decoder ReLU masks are applied in the dgrad epilogues; skip-connection gradients are
accumulated with TMA reduce-add."""
import os
import torch
import torch.distributed as dist
from torch import nn

from . import _lib as L
from . import ops

BF16 = torch.bfloat16
F32 = torch.float32

# the only launch kinds a builder may mark `side`: weight-gradient GEMMs, which only add into the gradient arena
_SIDE_KINDS = frozenset(("conv_wgrad", "convt_wgrad"))


class _Op:
    """one launch (or a tiny group) with its algorithmic cost, for the per-kernel breakdown in bench.py.  `side`: a
    weight-gradient launch that Plan._run_bwd forks onto the side stream (nothing later in the step reads its output)"""
    __slots__ = ("kind", "fn", "flops", "bytes", "desc", "side")

    def __init__(self, kind, fn, flops=0.0, nbytes=0.0, desc="", side=False):
        if side and kind not in _SIDE_KINDS:
            raise RuntimeError("plan error: a %s launch cannot run on the side stream" % kind)
        self.kind, self.fn, self.flops, self.bytes, self.desc = kind, fn, float(flops), float(nbytes), desc
        self.side = side

    def __call__(self):
        return self.fn()


def _nb(*tensors):
    return float(sum(t.numel() * t.element_size() for t in tensors if t is not None))


def _conv_desc(x, cout, k, s):
    """breakdown label of a k x k / stride s conv over x"""
    return "%d->%d k%d s%d @%dx%dx%d" % ((x.shape[3], cout, k, s) + tuple(x.shape[:3]))


def graph_capture(graph, dev):
    """torch.cuda.graph context on a HIGH-priority capture stream: the captured step's main chain runs at high priority
    while the backward's side stream (weight-gradient GEMMs, Adam segments, all-reduce launches) keeps the default low
    priority, so the block scheduler serves the critical path (data-gradient GEMMs + BatchNorm-backward) first and the
    side work, forked as soon as its operands exist (Plan._run_bwd), fills what is left."""
    return torch.cuda.graph(graph, stream=torch.cuda.Stream(device=dev, priority=-1))


class _OpList(list):
    """list of _Op; .add(kind, fn, flops, bytes, desc, side)"""

    def add(self, kind, fn, flops=0.0, nbytes=0.0, desc="", side=False):
        self.append(_Op(kind, fn, flops, nbytes, desc, side))


class _BN:
    """per-BatchNorm device state"""
    __slots__ = ("mod", "c", "stats", "scale", "shift", "mean", "invstd", "gamma", "beta", "dgamma", "dbeta", "tr",
                 "idx", "off", "app_dgamma", "app_dbeta", "g32_dgamma", "g32_dbeta")


class _ConvPart:
    """one conv + BatchNorm of a ResNet block, for per-unit tests: the state_dict prefixes of the conv and its
    BatchNorm, the conv's input x and output z, the BatchNorm output y, the _BN state and the backward's dz buffer.
    Training: y is None for the block's last conv and its downsample, whose BatchNorms the residual pass applies.
    Inference: the BatchNorm (and the residual, the ReLU) is folded into the conv epilogue, so y is z, the stored
    output, and dz stays None"""
    __slots__ = ("conv", "bn", "x", "z", "y", "state", "dz")

    def __init__(self, conv, bn, x, z, y, state):
        self.conv, self.bn, self.x, self.z, self.y, self.state, self.dz = conv, bn, x, z, y, state, None


class Plan:
    """What every launch plan shares: activation and gradient buffers, the BatchNorm units, the decoder blocks and the
    classifier tail, backward registration, the arena segments and execution.  A subclass per encoder family builds
    the network in _build() and names its three segment boundaries in _segment_bounds()."""

    def __init__(self, net, n, h, w, training):
        self.net, self.n, self.h, self.w, self.training = net, n, h, w, training
        self.dev = net._p32.device
        self.fwd_ops = _OpList()   # _Op launches, in order
        self.bwd_layers = []       # list of lists of closures (one list per forward unit), executed in reverse
        self.grad = {}             # id(activation) -> gradient buffer
        self.written = set()       # gradient buffers that already hold a contribution
        self._keep = []            # keeps tensors referenced by closures alive
        self._bns = []
        self._bwd_builders = []    # (tag, builder) per forward unit; run in REVERSE so store/accumulate modes follow run order
        self.units = []            # (kind, state_dict prefix, inputs, output) per forward unit, for per-unit parity tests
        self.dec_mid = {}          # id(decoder block output) -> the block's middle ConvRelu output, for the same tests
        self.block_parts = {}      # ResNet plans: id(block output) -> [_ConvPart], conv1 .. [downsample]
        self.stem_parts = {}       # ResNet plans: the stem's col, z0, a0, c1, bn0 (and dz0 when training; z0 is a0
        #                            when not: the inference stem folds its BatchNorm and ReLU into the GEMM)
        self.classifier_in = None  # the last ConvRelu's output, which the 1x1 classifier reads
        total_c = sum(m.num_features for m in net.modules() if isinstance(m, nn.BatchNorm2d))
        n_bn = sum(1 for m in net.modules() if isinstance(m, nn.BatchNorm2d))
        self._stats_arena = torch.zeros(2 * total_c, dtype=F32, device=self.dev)
        self._stats_used = 0
        self.graph_fwd = self.graph_bwd = None
        self._side = None
        # Synchronised BatchNorm (opt-in, MCB_SYNC_BN=1, one process per GPU): every BatchNorm normalises with the
        # statistics of the GLOBAL batch -- [sum, sum^2] all-reduced between the conv that produces them and the BN
        # apply pass, [dbeta, dgamma] all-reduced before the dz pass.  The default keeps the reference's DataParallel
        # semantics (per-replica statistics, src/models.py:65).  The collectives are issued from the plan, so they are
        # captured into the step's CUDA graphs with everything else.
        self.world = dist.get_world_size() if (dist.is_available() and dist.is_initialized()) else 1
        mode = os.environ.get("MCB_SYNC_BN", "0")
        self.sync_bn = training and self.world > 1 and mode in ("1", "2")
        # MCB_SYNC_BN=2: the per-BatchNorm exchange is a one-shot all-reduce over NVLink peer memory (csrc/sync.cu) instead
        # of a NCCL call: every rank pushes its partial sums into its peers' receive buffers (symmetric memory)
        self.sync_nvlink = self.sync_bn and mode == "2"
        self.bn_scale = self.world if self.sync_bn else 1
        if self.sync_nvlink:
            import torch.distributed._symmetric_memory as symm
            grp = dist.group.WORLD
            self.rank = dist.get_rank()

            def sym(n, dtype):
                t = symm.empty(n, dtype=dtype, device=self.dev)
                t.zero_()
                h = symm.rendezvous(t, grp)
                ptrs = torch.tensor([int(p) for p in h.buffer_ptrs], dtype=torch.int64, device=self.dev)
                self._keep.append(h)
                return t, ptrs
            # partial sums stay in LOCAL memory; every rank owns receive buffers [world][2 total_c] that its peers push into
            self._dstats_loc = torch.zeros(2 * total_c, dtype=F32, device=self.dev)      # [dbeta | dgamma] partial sums
            # (value, stamp) pairs: 2 floats per entry
            self._recv_stats, self._peer_recv_stats = sym(self.world * 2 * total_c * 2, F32)
            self._recv_dstats, self._peer_recv_dstats = sym(self.world * 2 * total_c * 2, F32)
            self._sync_stride = 2 * total_c
            self._gstats = torch.zeros(2 * total_c, dtype=F32, device=self.dev)    # global [sum, sum^2]
            self._gdstats = torch.zeros(2 * total_c, dtype=F32, device=self.dev)   # global [dbeta | dgamma]
            self._sync_step = torch.zeros(1, dtype=torch.int32, device=self.dev)
            self._n_bn = n_bn
            torch.cuda.synchronize()
            dist.barrier()
        self.bias_sum = {}         # id(conv+bias+ReLU output) -> its bias-gradient vector (fused into the consumer's dgrad)
        self.bias_fused = set()
        self.x_in = torch.zeros((n, 3, h, w), dtype=F32, device=self.dev)
        self.dlogits = torch.zeros((n, net.num_classes, h, w), dtype=F32, device=self.dev)
        self.logits = torch.zeros((n, net.num_classes, h, w), dtype=F32, device=self.dev)
        self._build()
        self.bwd_tags = []
        for tag, builder in reversed(self._bwd_builders):
            B = _OpList()
            builder(B)
            self.bwd_layers.append(B)
            self.bwd_tags.append(tag)
        self.launches_fwd = len(self.fwd_ops)
        self.launches_bwd = sum(len(l) for l in self.bwd_layers)
        # inference folds every BatchNorm into a per-channel affine: one launch refreshes all of them from the running
        # statistics, over rows [gamma, beta, running_mean, running_var, scale, shift, C]
        self._bn_tab = None
        if self._bns and not training:
            rows = [[b.gamma.data_ptr(), b.beta.data_ptr(), b.mod.running_mean.data_ptr(), b.mod.running_var.data_ptr(),
                     b.scale.data_ptr(), b.shift.data_ptr(), b.c] for b in self._bns]
            self._bn_tab = torch.tensor(rows, dtype=torch.int64, device=self.dev)

    def _build(self):
        raise NotImplementedError

    def _segment_bounds(self):
        """the family's three backward segment boundaries, deepest-first: [(bwd tag, first arena parameter)]"""
        raise NotImplementedError

    # ------------------------------------------------------------------------------------------ helpers
    def act(self, n, h, w, c):
        t = torch.zeros((n, h, w, c), dtype=BF16, device=self.dev)
        self._keep.append(t)
        return t

    def gbuf(self, a):
        g = self.grad.get(id(a))
        if g is None:
            g = torch.zeros_like(a)
            self.grad[id(a)] = g
            self._keep.append(g)
        return g

    def gmode(self, a):
        """-> accumulate flag for the next writer of grad(a); marks it written"""
        acc = id(a) in self.written
        self.written.add(id(a))
        return acc

    def on_backward(self, tag, builder):
        """register builder(B), which appends one forward unit's backward launches to B; `tag` names the unit's group
        for bwd_segments.  Inference plans have no backward."""
        if self.training:
            self._bwd_builders.append((tag, builder))

    def bn_state(self, mod):
        net = self.net
        b = _BN()
        b.mod, b.c = mod, mod.num_features
        c = b.c
        buf = torch.zeros(4 * c, dtype=F32, device=self.dev)
        self._keep.append(buf)
        b.idx, b.off = len(self._bns), self._stats_used
        b.stats = self._stats_arena[self._stats_used:self._stats_used + 2 * c]
        self._stats_used += 2 * c
        b.scale, b.shift, b.mean, b.invstd = buf[:c], buf[c:2 * c], buf[2 * c:3 * c], buf[3 * c:4 * c]
        b.gamma, b.beta = net._vec(mod.weight, net._p32), net._vec(mod.bias, net._p32)
        b.g32_dgamma, b.g32_dbeta = net._vec(mod.weight, net._g32), net._vec(mod.bias, net._g32)
        if self.sync_nvlink:
            # the reduction kernels accumulate this rank's partial sums in symmetric memory; the exchange writes the
            # global sums to local buffers (what the normalisation passes read) and global / world to the gradient slots
            b.dbeta, b.dgamma = self._dstats_loc[b.off:b.off + c], self._dstats_loc[b.off + c:b.off + 2 * c]
            b.app_dbeta, b.app_dgamma = self._gdstats[b.off:b.off + c], self._gdstats[b.off + c:b.off + 2 * c]
            tr_stats = self._gstats[b.off:b.off + 2 * c]
        else:
            b.dgamma, b.dbeta = b.g32_dgamma, b.g32_dbeta
            b.app_dgamma, b.app_dbeta = b.dgamma, b.dbeta
            tr_stats = b.stats
        b.tr = ops.make_bn_train(tr_stats, b.gamma, b.beta, mod.running_mean, mod.running_var, b.mean, b.invstd) \
            if self.training else None
        self._bns.append(b)
        return b

    # one conv (+BN) unit ------------------------------------------------------------------------------
    def conv_bn(self, x, conv, bnmod, relu, residual=None, res_bn=None, out=None):
        """z = conv(x); y = [relu](bn(z) [+ residual | + res_bn(residual_raw)]).  Returns (y, z, bn).  When `relu` is
        None the BN apply is deferred (the caller fuses it into a later residual pass) and y is None."""
        net = self.net
        k, s = conv.kernel_size[0], conv.stride[0]
        n, h, w, cin = x.shape
        cout = conv.out_channels
        z = self.act(n, h // s, w // s, cout)
        bn = self.bn_state(bnmod)
        w16 = net._packed(conv.weight, net._w16)
        F = self.fwd_ops
        cflops = 2.0 * z.numel() * cin * k * k
        desc = _conv_desc(x, cout, k, s)
        if self.training:
            F.add("conv_fwd", lambda: ops.conv_fwd(x, w16, k, s, stats=bn.stats, out=z), cflops, _nb(x, w16, z), desc)
            self.sync_stats(F, bn)
        else:
            # inference: BatchNorm is a per-channel affine known up front -> folded into the conv epilogue together with
            # the residual add and the ReLU; no pre-BN tensor is materialised (z IS the block output here)
            do_relu = bool(relu) if relu is not None else False
            F.add("conv_fwd", lambda: ops.conv_fwd(x, w16, k, s, bias=bn.shift, relu=do_relu, scale=bn.scale,
                                                   residual=residual, out=z), cflops, _nb(x, w16, z, residual), desc)
            return z, z, bn
        if relu is None:
            return None, z, bn
        y = out if out is not None else self.act(*z.shape)
        self.bn_apply_op(z, bn, y, relu, residual, res_bn)
        return y, z, bn

    def bn_apply_op(self, z, bn, y, relu, residual=None, res_bn=None):
        """BN (+residual [+ its BN]) + ReLU in one pass; training mode folds the statistics finalisation in"""
        F = self.fwd_ops
        if self.training:
            rtr = res_bn.tr if res_bn is not None else None
            F.add("bn_apply", lambda: ops.bn_train_apply(z, bn.tr, y, relu, residual, rtr, BN_MOMENTUM, BN_EPS,
                                                         self.bn_scale), 0, _nb(z, y, residual))
        elif res_bn is not None:
            F.add("bn_apply", lambda: ops.bn_apply(z, bn.scale, bn.shift, y, relu, residual, res_bn.scale,
                                                   res_bn.shift), 0, _nb(z, y, residual))
        else:
            F.add("bn_apply", lambda: ops.bn_apply(z, bn.scale, bn.shift, y, relu, residual), 0, _nb(z, y, residual))

    def sync_stats(self, F, bn):
        """SyncBN forward: sum the per-rank [sum, sum^2] before the BN apply pass reads them"""
        if self.sync_nvlink:
            F.add("bn_exchange", lambda: L.fcall(
                "mcb_sync_exchange", self._stats_arena.data_ptr(), self._peer_recv_stats.data_ptr(), self.rank, self.world,
                self._sync_stride, bn.off, 2 * bn.c, self._sync_step.data_ptr(), self._gstats[bn.off:].data_ptr(), None,
                None, 0, 0.0))
        elif self.sync_bn:
            F.add("bn_allreduce", lambda: dist.all_reduce(bn.stats))

    def sync_bn_grads(self, B, bn):
        """SyncBN backward: dz needs the GLOBAL dbeta / dgamma.  They are the parameter-gradient slots themselves, so
        after this they hold the global sums on every rank (FusedTrainStep divides them by the world size before the
        arena-wide gradient all-reduce adds the ranks up again)."""
        if self.sync_nvlink:
            B.add("bn_exchange", lambda: L.fcall(
                "mcb_sync_exchange", self._dstats_loc.data_ptr(), self._peer_recv_dstats.data_ptr(), self.rank, self.world,
                self._sync_stride, bn.off, 2 * bn.c, self._sync_step.data_ptr(), self._gdstats[bn.off:].data_ptr(),
                bn.g32_dbeta.data_ptr(), bn.g32_dgamma.data_ptr(), bn.c, 1.0 / self.world))
        elif self.sync_bn:
            g32 = self.net._g32
            lo = (bn.dgamma.data_ptr() - g32.data_ptr()) // 4
            hi = (bn.dbeta.data_ptr() - g32.data_ptr()) // 4
            if hi == lo + bn.c:       # gamma and beta slots are adjacent: one collective
                both = g32[lo:lo + 2 * bn.c]
                B.add("bn_allreduce", lambda: dist.all_reduce(both))
            else:
                B.add("bn_allreduce", lambda: (dist.all_reduce(bn.dgamma), dist.all_reduce(bn.dbeta)))

    def bn_grad_slices(self):
        """views of every BatchNorm weight/bias gradient in the arena (see sync_bn_grads)"""
        return [t for b in self._bns for t in (b.dgamma, b.dbeta)]

    def conv_unit_backward(self, B, dy, ymask, z, bn, conv, x, g_out=None, g_out_acc=False, reduced=False):
        """backward of y = relu(bn(conv(x)) [+ r]) given dy = dL/dy: BN reductions + dz, wgrad, dgrad into grad(x).
        g_out receives g = dy*(y>0) for a residual branch."""
        net = self.net
        k, s = conv.kernel_size[0], conv.stride[0]
        dz = self.act(*z.shape)
        gw = net._packed(conv.weight, net._g32)
        if not reduced:  # else: the dgrad that produced dy already accumulated dbeta / dgamma in its epilogue
            B.add("bn_bwd_reduce", lambda: ops.bn_bwd_reduce(dy, ymask, z, bn.mean, bn.invstd, bn.dbeta, bn.dgamma),
                  0, _nb(dy, ymask, z))
        self.sync_bn_grads(B, bn)
        B.add("bn_bwd_apply", lambda: ops.bn_bwd_apply(dy, ymask, z, bn.mean, bn.invstd, bn.gamma, bn.app_dbeta,
                                                      bn.app_dgamma, dz, g_out, g_out_acc, self.bn_scale), 0,
              _nb(dy, ymask, z, dz, g_out))
        B.add("conv_wgrad", lambda: ops.conv_wgrad(dz, x, gw, k, s), 2.0 * dz.numel() * x.shape[3] * k * k,
              _nb(dz, x, gw), _conv_desc(x, dz.shape[3], k, s), side=True)
        return dz

    def dgrad_into(self, B, dz, conv, x, relu_mask=None, ci_off=0, bn_reduce=None):
        """grad(x) (+)= dgrad(dz); bn_reduce = (z, bn): fuse that BatchNorm's backward reductions into the epilogue"""
        net = self.net
        k, s = conv.kernel_size[0], conv.stride[0]
        w16 = net._packed(conv.weight, net._w16)
        gx = self.gbuf(x)
        acc = self.gmode(x)
        hw = (x.shape[1], x.shape[2])
        cin = x.shape[3]
        if acc and relu_mask is not None:
            raise RuntimeError("plan error: masked dgrad cannot accumulate")
        csum = None
        if relu_mask is x and id(x) in self.bias_sum:
            csum = self.bias_sum[id(x)]      # x = relu(conv(.) + b): its bias gradient is the channel sum of grad(x)
            self.bias_fused.add(id(x))
        red = None
        if bn_reduce is not None:
            zz, bb = bn_reduce
            red = (zz, bb.mean, bb.invstd, bb.gamma, bb.beta, bb.dbeta, bb.dgamma)
            relu_mask = None  # recomputed from z in the epilogue
        B.add("conv_dgrad", lambda: ops.conv_dgrad(dz, w16, k, s, hw, cin=cin, ci_off=ci_off, relu_mask=relu_mask,
                                                   accumulate=acc, out=gx, bn_reduce=red, channel_sum=csum),
              2.0 * dz.numel() * cin * k * k,
              _nb(dz, gx, relu_mask) + (_nb(gx) if acc else 0) + 2.0 * k * k * dz.shape[3] * cin,
              "%d<-%d k%d s%d @%dx%dx%d%s" % (cin, dz.shape[3], k, s, x.shape[0], x.shape[1], x.shape[2],
                                              " acc" if acc else ""))

    # ------------------------------------------------------------------------------------------ decoder
    def _conv_relu(self, x1, skip, conv, label):
        """ConvRelu over cat[x1, skip] (src/unet_models.py:25-34): relu(conv3x3(.) + b), the concat fused into the
        GEMM; `label`: give its launch a breakdown label"""
        net = self.net
        n, h, w, c1 = x1.shape
        cout = conv.out_channels
        w16 = net._packed(conv.weight, net._w16)
        b = net._vec(conv.bias, net._p32)
        y = self.act(n, h, w, cout)
        ctot = c1 + (skip.shape[3] if skip is not None else 0)
        self.fwd_ops.add("conv_fwd", lambda: ops.conv_fwd(x1, w16, 3, 1, bias=b, relu=True, x2=skip, out=y),
                         2.0 * y.numel() * ctot * 9, _nb(x1, skip, w16, y),
                         "dec %d->%d k3 @%dx%dx%d" % (ctot, cout, n, h, w) if label else "")
        return y

    def _conv_relu_backward(self, B, g, conv, x1, skip, x1_relu, label, side):
        """weight and data gradients of _conv_relu given g, the gradient of its output with the ReLU mask applied.
        x1_relu: x1 is a ReLU output (its mask rides in the dgrad epilogue); the skip's mask is applied by its owner.
        `side`: the weight-gradient GEMMs go to the side stream"""
        gw = self.net._packed(conv.weight, self.net._g32)
        n, h, w, cout = g.shape
        c1 = x1.shape[3]
        srcs = [(x1, 0, "dec")] if skip is None else [(x1, 0, "dec"), (skip, c1, "dec-skip")]
        for x, ci_off, name in srcs:
            B.add("conv_wgrad", lambda x=x, ci_off=ci_off: ops.conv_wgrad(g, x, gw, 3, 1, ci_off=ci_off),
                  2.0 * g.numel() * x.shape[3] * 9, _nb(g, x),
                  "%s %d->%d k3 @%dx%dx%d" % (name, x.shape[3], cout, n, h, w) if label else "", side)
        self.dgrad_into(B, g, conv, x1, relu_mask=x1 if x1_relu else None)
        if skip is not None:
            self.dgrad_into(B, g, conv, skip, ci_off=c1)

    def _decoder(self, x1, skip, block, pool_input=False):
        """DecoderBlockV2 / DecoderBlock: relu(conv3x3(cat[x1, skip]) + b) -> relu(convT(.) + b) with the 4x4 or the 3x3
        (output_padding 1) stride-2 transposed conv   (src/unet_models.py:42-53,136-141)"""
        net = self.net
        conv, deconv = block.block[0].conv, block.block[1]
        mid = self._conv_relu(x1, skip, conv, label=True)
        n, h, w, cmid = mid.shape
        cout = deconv.out_channels
        kt = deconv.kernel_size[0]
        wt16 = net._packed(deconv.weight, net._w16)
        b2 = net._vec(deconv.bias, net._p32)
        out = self.act(n, 2 * h, 2 * w, cout)
        self.dec_mid[id(out)] = mid
        self.bias_sum[id(out)] = net._vec(deconv.bias, net._g32)
        ft = 2.0 * mid.numel() * cout * kt * kt
        dd = "%d->%d @%dx%dx%d" % (cmid, cout, n, h, w)
        self.fwd_ops.add("convt_fwd", lambda: ops.convt_fwd(mid, wt16, bias=b2, relu=True, out=out), ft,
                         _nb(mid, wt16, out), dd)

        def build_dec(B):
            g_out = self.gbuf(out)   # already masked by out's ReLU (the consumer's dgrad epilogue did it)
            g_mid = self.gbuf(mid)
            gwt = net._packed(deconv.weight, net._g32)
            gb2 = net._vec(deconv.bias, net._g32)
            gb1 = net._vec(conv.bias, net._g32)
            if id(out) not in self.bias_fused:   # else: summed in the epilogue of the dgrad that produced g_out
                B.add("channel_sum", lambda: ops.channel_sum(g_out, gb2), 0, _nb(g_out))
            B.add("convt_wgrad", lambda: ops.convt_wgrad(g_out, mid, gwt), ft, _nb(g_out, mid, gwt), dd, side=True)
            B.add("convt_dgrad", lambda: ops.convt_dgrad(g_out, wt16, relu_mask=mid, out=g_mid, channel_sum=gb1), ft,
                  _nb(g_out, wt16, mid, g_mid), dd)
            # x1 is a decoder ReLU output unless it is the centre's max-pool output
            self._conv_relu_backward(B, g_mid, conv, x1, skip, not pool_input, label=True, side=True)
        self.on_backward("decoder", build_dec)
        return out

    def _classifier(self, x1, skip, conv_relu, label, side):
        """the last ConvRelu over cat[x1, skip] and the 1x1 classifier into self.logits, whose backward also applies the
        ConvRelu's ReLU mask.  `label` / `side`: breakdown labels and side-stream placement of its conv launches"""
        net = self.net
        conv = conv_relu.conv
        y = self._conv_relu(x1, skip, conv, label)
        self.classifier_in = y
        fw, fb = net._vec(net.final.weight, net._p32), net._vec(net.final.bias, net._p32)
        self.fwd_ops.add("final_conv", lambda: ops.final_conv_fwd(y, fw, fb, self.logits),
                         2.0 * self.logits.numel() * 32, _nb(y, self.logits))

        def build_head(B):
            g = self.gbuf(y)
            gfw, gfb = net._vec(net.final.weight, net._g32), net._vec(net.final.bias, net._g32)
            B.add("final_conv", lambda: ops.final_conv_bwd(y, fw, self.dlogits, g, gfw, gfb),
                  4.0 * self.logits.numel() * 32, _nb(y, self.dlogits, g))
            gb = net._vec(conv.bias, net._g32)
            B.add("channel_sum", lambda: ops.channel_sum(g, gb), 0, _nb(g))
            self._conv_relu_backward(B, g, conv, x1, skip, True, label, side)
        self.on_backward("decoder", build_head)
        return y

    # ------------------------------------------------------------------------------------------ execution
    def _run_fwd(self):
        if self._bn_tab is not None:
            L.fcall("mcb_bn_eval_params_batched", self._bn_tab.data_ptr(), len(self._bns), max(b.c for b in self._bns),
                    BN_EPS)
        if self.training:
            if self.sync_nvlink:
                L.fcall("mcb_sync_step_bump", self._sync_step.data_ptr())
            if self._stats_arena.numel():
                L.zero(self._stats_arena)
        for op in self.fwd_ops:
            op()

    def _run_bwd(self, hooks=None):
        """all backward layers in execution (reverse-forward) order, after zeroing the gradient arena.
        hooks = {layer_index: fn}: fn() runs ON THE SIDE STREAM once every launch of the layers before `layer_index`
        (main chain and weight-gradient GEMMs) is ordered before it -- used for per-segment optimizer updates and
        all-reduces that overlap the rest of the backward pass."""
        L.zero(self.net._g32)
        if self.sync_nvlink:
            L.zero(self._dstats_loc)
        # Weight-gradient launches marked `side` are leaves of the backward graph (they only add into the gradient
        # arena): each goes to the low-priority side stream, forked right after its producer and joined at the end, so
        # the tensor-core-bound wgrad GEMMs overlap the HBM-bound BatchNorm-backward kernels of the layers below instead
        # of queueing behind them, and the high-priority main chain (graph_capture) is served first.
        # (No buffer is recycled inside a step, so the only hazards are the recorded producer -> consumer edges.)
        main = torch.cuda.current_stream()
        if self._side is None:
            self._side = torch.cuda.Stream(device=self.dev)
        forked = False

        def on_side(fn):
            nonlocal forked
            ev = torch.cuda.Event()
            ev.record(main)
            self._side.wait_event(ev)
            with torch.cuda.stream(self._side):
                fn()
            forked = True

        for li, layer in enumerate(self.bwd_layers):
            if hooks and li in hooks:
                on_side(hooks[li])
            for op in layer:
                if op.side:
                    on_side(op)
                else:
                    op()
        if hooks and len(self.bwd_layers) in hooks:
            on_side(hooks[len(self.bwd_layers)])
        if forked:
            ev = torch.cuda.Event()
            ev.record(self._side)
            main.wait_event(ev)

    def bwd_segments(self):
        """split points for overlapping the gradient all-reduce / the Adam update with the backward pass, at the
        family's _segment_bounds (ResNets: [decoder | layer4 | layer3 | rest]).
        -> [(first_layer, last_layer, arena_lo, arena_hi)], the arena range is complete once the segment has run
        (layer3's 23 blocks reduce while layer2 / layer1 / stem still run)"""
        net = self.net
        off = {name: net._slots[id(p)].off for name, p, _ in net._arena_params()}
        segs = []
        first, hi = 0, net._p32.numel()
        for tag, param in self._segment_bounds():
            last = max(i for i, t in enumerate(self.bwd_tags) if t == tag) + 1
            segs.append((first, last, off[param], hi))
            first, hi = last, off[param]
        return segs + [(first, len(self.bwd_tags), 0, hi)]

    def forward(self, x):
        self.x_in.copy_(x)
        if self.graph_fwd is None:
            self._run_fwd()  # eager warm-up (sets kernel attributes, validates arguments)
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with graph_capture(g, self.dev):
                self._run_fwd()
            self.graph_fwd = g
            return self.logits
        self.graph_fwd.replay()
        return self.logits

    def backward(self, dlogits):
        self.dlogits.copy_(dlogits)
        if self.graph_bwd is None:
            self._run_bwd()
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with graph_capture(g, self.dev):
                self._run_bwd()
            self.graph_bwd = g
            return
        self.graph_bwd.replay()


class ResNetPlan(Plan):
    """UNetResNet / AlbuNet (src/unet_models.py:315-403): 7x7 stem, torchvision BasicBlock / Bottleneck stages, the
    DecoderBlockV2 decoder, dec0 and the classifier"""

    def _segment_bounds(self):
        return [("decoder", "center.block.0.conv.weight"), ("layer4", "encoder.layer4.0.conv1.weight"),
                ("layer3", "encoder.layer3.0.conv1.weight")]

    def _build(self):
        net, n, h, w = self.net, self.n, self.h, self.w
        F = self.fwd_ops
        enc = net.encoder

        # ---- stem: 7x7/s2 conv as im2col + GEMM, BN, ReLU, 2x2 max-pool (src/unet_models.py:360-363)
        col = self.act(n, h // 2, w // 2, 192)
        stem_w16 = torch.zeros((1, 64, 192), dtype=BF16, device=self.dev)
        self._keep.append(stem_w16)
        stem_master = net._vec(enc.conv1.weight, net._p32)
        F.add("stem_im2col", lambda: ops.stem_im2col(self.x_in, col), 0, _nb(self.x_in, col))
        F.add("misc", lambda: ops.stem_pack_weight(stem_master, stem_w16))
        sflops = 2.0 * n * (h // 2) * (w // 2) * 64 * 147
        z0 = self.act(n, h // 2, w // 2, 64)
        bn0 = self.bn_state(enc.bn1)
        if self.training:
            F.add("conv_fwd", lambda: ops.conv_fwd(col, stem_w16, 1, 1, stats=bn0.stats, out=z0), sflops, _nb(col, z0))
            self.sync_stats(F, bn0)
            a0 = self.act(*z0.shape)
            self.bn_apply_op(z0, bn0, a0, True)
        else:
            F.add("conv_fwd", lambda: ops.conv_fwd(col, stem_w16, 1, 1, bias=bn0.shift, relu=True, scale=bn0.scale,
                                                   out=z0), sflops, _nb(col, z0))
            a0 = z0
        c1 = self.act(n, h // 4, w // 4, 64)
        F.add("maxpool", lambda: ops.maxpool2_fwd(a0, c1), 0, _nb(a0, c1))
        self.stem_parts.update(col=col, z0=z0, a0=a0, c1=c1, bn0=bn0)

        def build_stem(B):
            d_a0 = self.gbuf(a0)
            d_c1 = self.gbuf(c1)
            dz0 = self.act(*z0.shape)
            self.stem_parts["dz0"] = dz0
            stem_gw = torch.zeros((1, 64, 192), dtype=F32, device=self.dev)
            self._keep.append(stem_gw)
            stem_g = net._vec(enc.conv1.weight, net._g32)
            B.add("maxpool", lambda: ops.maxpool2_bwd(a0, d_c1, d_a0, False), 0, _nb(a0, d_c1, d_a0))
            B.add("bn_bwd_reduce", lambda: ops.bn_bwd_reduce(d_a0, a0, z0, bn0.mean, bn0.invstd, bn0.dbeta,
                                                            bn0.dgamma), 0, _nb(d_a0, a0, z0))
            self.sync_bn_grads(B, bn0)
            B.add("bn_bwd_apply", lambda: ops.bn_bwd_apply(d_a0, a0, z0, bn0.mean, bn0.invstd, bn0.gamma,
                                                          bn0.app_dbeta, bn0.app_dgamma, dz0, None, False,
                                                          self.bn_scale),
                  0, _nb(d_a0, a0, z0, dz0))
            B.add("misc", lambda: L.zero(stem_gw))
            # on the main stream: the unpack that follows reads stem_gw
            B.add("conv_wgrad", lambda: ops.conv_wgrad(dz0, col, stem_gw, 1, 1), sflops, _nb(dz0, col))
            B.add("misc", lambda: ops.stem_unpack_wgrad(stem_gw, stem_g))
        self.on_backward("stem", build_stem)

        # ---- encoder stages (torchvision BasicBlock / Bottleneck)
        x = c1
        skips = []
        for li, layer in enumerate((enc.layer1, enc.layer2, enc.layer3, enc.layer4)):
            for bi, blk in enumerate(layer):
                xin = x
                prefix = "encoder.layer%d.%d" % (li + 1, bi)
                x = self._res_block(x, blk, "layer%d" % (li + 1), prefix)
                self.units.append(("block", prefix, (xin,), x))
            skips.append(x)
        c2, c3, c4, c5 = skips

        # ---- centre + decoder (src/unet_models.py:373-403)
        pool = self.act(n, c5.shape[1] // 2, c5.shape[2] // 2, c5.shape[3])
        F.add("maxpool", lambda: ops.maxpool2_fwd(c5, pool), 0, _nb(c5, pool))

        def build_pool(B):
            d_pool, d_c5 = self.gbuf(pool), self.gbuf(c5)
            acc = self.gmode(c5)  # dec5's skip dgrad ran first -> accumulate
            B.add("maxpool", lambda: ops.maxpool2_bwd(c5, d_pool, d_c5, acc), 0, _nb(c5, d_pool, d_c5))
        self.on_backward("decoder", build_pool)
        center = self._decoder(pool, None, net.center, pool_input=True)
        d5 = self._decoder(center, c5, net.dec5)
        d4 = self._decoder(d5, c4, net.dec4)
        d3 = self._decoder(d4, c3, net.dec3)
        d2 = self._decoder(d3, c2, net.dec2)
        d1 = self._decoder(d2, None, net.dec1)
        self.units += [("decoder", "center", (pool,), center), ("decoder", "dec5", (center, c5), d5),
                       ("decoder", "dec4", (d5, c4), d4), ("decoder", "dec3", (d4, c3), d3),
                       ("decoder", "dec2", (d3, c2), d2), ("decoder", "dec1", (d2,), d1)]
        # dec0 = ConvRelu(32, 32): unlabelled, its weight gradient on the main stream
        self._classifier(d1, None, net.dec0, label=False, side=False)

    def _res_block(self, x, blk, tag, prefix):
        """torchvision BasicBlock / Bottleneck forward + backward plan; `prefix`: the block's state_dict prefix"""
        is_bottleneck = hasattr(blk, "conv3")
        convs = [(blk.conv1, blk.bn1), (blk.conv2, blk.bn2)] + ([(blk.conv3, blk.bn3)] if is_bottleneck else [])
        names = [("%s.conv%d" % (prefix, i), "%s.bn%d" % (prefix, i)) for i in range(1, len(convs) + 1)]
        if not self.training:
            # every conv's output is its folded BatchNorm's output: the parts record it as both z and y
            parts = []
            cur = x
            for (conv, bnm), (cname, bname) in zip(convs[:-1], names):
                y, _, bn = self.conv_bn(cur, conv, bnm, True)
                parts.append(_ConvPart(cname, bname, cur, y, y, bn))
                cur = y
            ident = x
            down = None
            if blk.downsample is not None:
                ident, _, bnd = self.conv_bn(x, blk.downsample[0], blk.downsample[1], False)
                down = _ConvPart(prefix + ".downsample.0", prefix + ".downsample.1", x, ident, ident, bnd)
            out, _, bnl = self.conv_bn(cur, convs[-1][0], convs[-1][1], True, residual=ident)
            parts.append(_ConvPart(names[-1][0], names[-1][1], cur, out, out, bnl))
            self.block_parts[id(out)] = parts + ([down] if down is not None else [])
            return out
        units = []
        parts = []
        cur = x
        for (conv, bnm), (cname, bname) in zip(convs[:-1], names):
            y, z, bn = self.conv_bn(cur, conv, bnm, True)
            units.append((conv, cur, y, z, bn))
            parts.append(_ConvPart(cname, bname, cur, z, y, bn))
            cur = y
        conv_l, bn_l = convs[-1]
        _, z_l, bnl = self.conv_bn(cur, conv_l, bn_l, None)
        parts.append(_ConvPart(names[-1][0], names[-1][1], cur, z_l, None, bnl))
        out = self.act(*z_l.shape)
        if blk.downsample is not None:
            dconv, dbnm = blk.downsample[0], blk.downsample[1]
            _, zd, bnd = self.conv_bn(x, dconv, dbnm, None)
            parts.append(_ConvPart(prefix + ".downsample.0", prefix + ".downsample.1", x, zd, None, bnd))
            self.bn_apply_op(z_l, bnl, out, True, zd, bnd)
        else:
            self.bn_apply_op(z_l, bnl, out, True, x)
        last_in = cur
        self.block_parts[id(out)] = parts

        def build_block(B):
            d_out = self.gbuf(out)
            if blk.downsample is None:
                # identity branch: grad(x) (+)= g = d_out * (out > 0), emitted by the last BN's backward pass
                gx = self.gbuf(x)
                acc = self.gmode(x)
                dz_l = self.conv_unit_backward(B, d_out, out, z_l, bnl, conv_l, last_in, g_out=gx, g_out_acc=acc)
            else:
                dz_l = self.conv_unit_backward(B, d_out, out, z_l, bnl, conv_l, last_in)
            parts[len(units)].dz = dz_l
            # walk back through the inner units
            dz = dz_l
            conv_next = conv_l
            for i, (conv, xin, y, z, bn) in reversed(list(enumerate(units))):
                # y has a single consumer: its ReLU mask and its BN's backward reductions ride in the dgrad epilogue
                self.dgrad_into(B, dz, conv_next, y, bn_reduce=(z, bn))
                dz = self.conv_unit_backward(B, self.gbuf(y), None, z, bn, conv, xin, reduced=True)
                parts[i].dz = dz
                conv_next = conv
            self.dgrad_into(B, dz, conv_next, x)
            if blk.downsample is not None:
                dzd = self.conv_unit_backward(B, d_out, out, zd, bnd, dconv, x)
                parts[-1].dz = dzd
                self.dgrad_into(B, dzd, dconv, x)
        self.on_backward(tag, build_block)
        return out


class VGGPlan(Plan):
    """UNet11 / UNetVGG16 (src/unet_models.py:89-106, :296-312): five stages of conv + bias + ReLU units, each stage
    output pooled and concatenated into the decoder; no BatchNorm.  Backward: the decoder runs first and stores the
    skip segment's data gradient of every stage output; the pool backward adds the pooled path, applies the ReLU
    mask and sums the bias gradient (maxpool2_bwd_skip_relu).  Units inside a stage have one consumer: their mask
    and bias gradient ride in the next conv's dgrad epilogue."""

    def _segment_bounds(self):
        stages = self.net._stages
        return [("decoder", "center.block.0.conv.weight"), ("conv5", "encoder.%d.weight" % stages[4][0]),
                ("conv4", "encoder.%d.weight" % stages[3][0])]

    def _build(self):
        net = self.net
        enc = net.encoder
        skips = []
        x = None
        for si, stage in enumerate(net._stages):
            tag = "conv%d" % (si + 1)
            for idx in stage:
                xin = x
                x = self._input_unit(enc[idx], tag) if xin is None else self._unit(xin, enc[idx], tag)
                self.units.append(("conv", "encoder.%d" % idx, () if xin is None else (xin,), x))
            skips.append(x)
            x = self._pool(x, tag)
        c1, c2, c3, c4, c5 = skips
        # ---- decoder (src/unet_models.py:99-105, :303-310)
        center = self._decoder(x, None, net.center, pool_input=True)
        d5 = self._decoder(center, c5, net.dec5)
        d4 = self._decoder(d5, c4, net.dec4)
        d3 = self._decoder(d4, c3, net.dec3)
        d2 = self._decoder(d3, c2, net.dec2)
        self.units += [("decoder", "center", (x,), center), ("decoder", "dec5", (center, c5), d5),
                       ("decoder", "dec4", (d5, c4), d4), ("decoder", "dec3", (d4, c3), d3),
                       ("decoder", "dec2", (d3, c2), d2)]
        # dec1 = ConvRelu(32 + 64, 32) over cat[dec2, conv1]
        d1 = self._classifier(d2, c1, net.dec1, label=True, side=True)
        self.units.append(("decoder", "dec1", (d2, c1), d1))

    def _input_unit(self, conv, tag):
        """encoder.0 = Conv2d(3, 64, 3, padding 1) + ReLU on the full-resolution image: im2col (27 of 32 columns) + a
        1x1 GEMM with bias and ReLU; the weight gradient is the 1x1 wgrad, unpacked into the master slot"""
        net, n, h, w = self.net, self.n, self.h, self.w
        F = self.fwd_ops
        cout = conv.out_channels
        col = self.act(n, h, w, 32)
        w16 = torch.zeros((1, cout, 32), dtype=BF16, device=self.dev)
        self._keep.append(w16)
        master = net._vec(conv.weight, net._p32)
        b = net._vec(conv.bias, net._p32)
        y = self.act(n, h, w, cout)
        fl = 2.0 * n * h * w * cout * 27     # the real 27-wide reduction, as the reference counts it
        desc = "3->%d k3 (im2col) @%dx%dx%d" % (cout, n, h, w)
        F.add("im2col", lambda: ops.vgg_input_im2col(self.x_in, col), 0, _nb(self.x_in, col))
        F.add("misc", lambda: ops.vgg_input_pack_weight(master, w16))
        F.add("conv_fwd", lambda: ops.conv_fwd(col, w16, 1, 1, bias=b, relu=True, out=y), fl, _nb(col, y), desc)
        self.bias_sum[id(y)] = net._vec(conv.bias, net._g32)

        def build_input(B):
            g = self.gbuf(y)       # complete, masked, bias gradient summed (by its consumer)
            gw = torch.zeros((1, cout, 32), dtype=F32, device=self.dev)
            self._keep.append(gw)
            g_slot = net._vec(conv.weight, net._g32)
            B.add("misc", lambda: L.zero(gw))
            # on the main stream, in order with the zeroing and the unpack (like the ResNet stem)
            B.add("conv_wgrad", lambda: ops.conv_wgrad(g, col, gw, 1, 1), fl, _nb(g, col))
            B.add("misc", lambda: ops.vgg_input_unpack_wgrad(gw, g_slot))
        self.on_backward(tag, build_input)
        return y

    def _unit(self, x, conv, tag):
        """y = relu(conv3x3(x) + b).  x is a pool output (gradient stored plainly) or the previous unit's output (its
        ReLU mask and bias gradient fused into this unit's dgrad epilogue)"""
        net = self.net
        n, h, w, cin = x.shape
        cout = conv.out_channels
        w16 = net._packed(conv.weight, net._w16)
        b = net._vec(conv.bias, net._p32)
        y = self.act(n, h, w, cout)
        fl = 2.0 * y.numel() * cin * 9
        desc = _conv_desc(x, cout, 3, 1)
        self.fwd_ops.add("conv_fwd", lambda: ops.conv_fwd(x, w16, 3, 1, bias=b, relu=True, out=y), fl, _nb(x, w16, y),
                         desc)
        x_is_unit = id(x) in self.bias_sum
        self.bias_sum[id(y)] = net._vec(conv.bias, net._g32)

        def build_unit(B):
            g = self.gbuf(y)
            gw = net._packed(conv.weight, net._g32)
            B.add("conv_wgrad", lambda: ops.conv_wgrad(g, x, gw, 3, 1), fl, _nb(g, x, gw), desc, side=True)
            self.dgrad_into(B, g, conv, x, relu_mask=x if x_is_unit else None)
        self.on_backward(tag, build_unit)
        return y

    def _pool(self, y, tag):
        """2x2 max-pool of a stage output y; its backward completes grad(y) (see the class docstring)"""
        n, h, w, c = y.shape
        p = self.act(n, h // 2, w // 2, c)
        self.fwd_ops.add("maxpool", lambda: ops.maxpool2_fwd(y, p), 0, _nb(y, p))
        gb = self.bias_sum[id(y)]

        def build_pool(B):
            if id(y) not in self.written:
                raise RuntimeError("plan error: the skip gradient of a VGG stage output must be stored first")
            d_p, g = self.gbuf(p), self.gbuf(y)
            self.bias_fused.add(id(y))
            B.add("maxpool", lambda: ops.maxpool2_bwd_skip_relu(y, d_p, g, gb), 0, _nb(y, d_p, g, g))
        self.on_backward(tag, build_pool)
        return p


BN_MOMENTUM = 0.1
BN_EPS = 1e-5


class UNetFunction(torch.autograd.Function):
    """autograd bridge: logits = UNet(x); backward fills the gradient arena and hands its views to the parameters.
    Limitation (differs from torch): the arena is zeroed by every backward pass, so a SECOND backward() before
    optimizer.step() / zero_grad() replaces the gradients instead of accumulating into them -- the reference's
    _fit_loop (one backward per step, src/steps/pytorch/models.py:105-111) never does that; gradient accumulation
    over micro-batches needs the fused train step to grow an accumulate flag."""

    @staticmethod
    def forward(ctx, x, net, plan, *params):
        net.refresh_operands()
        logits = plan.forward(x)
        ctx.net, ctx.plan = net, plan
        return logits.clone()

    @staticmethod
    def backward(ctx, dlogits):
        net, plan = ctx.net, ctx.plan
        plan.backward(dlogits.contiguous())
        for p, gview in net.grad_views():
            if p.grad is None:
                p.grad = gview
            elif p.grad.data_ptr() != gview.data_ptr():
                p.grad.add_(gview)
        return (None, None, None) + tuple(None for _ in ctx.needs_input_grad[3:])
