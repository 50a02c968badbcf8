"""Static launch plans for UNetResNet: every kernel launch of one forward (and its backward) over preallocated
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


class _Op:
    """one launch (or a tiny group) with its algorithmic cost, for the per-kernel breakdown in bench.py"""
    __slots__ = ("kind", "fn", "flops", "bytes", "desc")

    def __init__(self, kind, fn, flops=0.0, nbytes=0.0, desc=""):
        self.kind, self.fn, self.flops, self.bytes, self.desc = kind, fn, float(flops), float(nbytes), desc

    def __call__(self):
        return self.fn()


def _nb(*tensors):
    return float(sum(t.numel() * t.element_size() for t in tensors if t is not None))


_SIDE_KINDS = frozenset(("conv_wgrad", "convt_wgrad"))


def stream_priority_enabled():
    """MCB_STREAM_PRIORITY (default 1): the captured step's main chain runs on a HIGH-priority stream while the backward's
    side stream (weight-gradient GEMMs, Adam segments, all-reduce launches) keeps the default low priority, so the block
    scheduler serves the critical path (data-gradient GEMMs + BatchNorm-backward) first and the side work fills what is
    left, together with launching every weight-gradient GEMM as soon as its operands exist (no deferral)."""
    return os.environ.get("MCB_STREAM_PRIORITY", "1") == "1"


def graph_capture(graph, dev):
    """torch.cuda.graph context on the high-priority capture stream (see stream_priority_enabled)"""
    if stream_priority_enabled():
        return torch.cuda.graph(graph, stream=torch.cuda.Stream(device=dev, priority=-1))
    return torch.cuda.graph(graph)


class _OpList(list):
    """list of _Op; .add(kind, fn, flops, bytes)"""

    # profiling aid: MCB_KNOCKOUT="kind,kind" drops those launches from the plan so that the step-time
    # difference gives their in-graph cost (results are garbage; never set outside profiling)
    _knockout = frozenset(k for k in os.environ.get("MCB_KNOCKOUT", "").split(",") if k)

    def add(self, kind, fn, flops=0.0, nbytes=0.0, desc=""):
        if kind in self._knockout:
            return
        self.append(_Op(kind, fn, flops, nbytes, desc))


class _BN:
    """per-BatchNorm device state"""
    __slots__ = ("mod", "c", "stats", "scale", "shift", "mean", "invstd", "gamma", "beta", "dgamma", "dbeta", "tr",
                 "idx", "off", "app_dgamma", "app_dbeta", "g32_dgamma", "g32_dbeta")


class Plan:
    def __init__(self, net, n, h, w, training):
        self.net, self.n, self.h, self.w, self.training = net, n, h, w, training
        self.dev = net._p32.device
        self.fwd_ops = _OpList()   # _Op launches, in order
        self.bwd_layers = []       # list of lists of closures (one list per forward unit), executed in reverse
        self.grad = {}             # id(activation) -> gradient buffer
        self.written = set()       # gradient buffers that already hold a contribution
        self._keep = []            # keeps tensors referenced by closures alive
        self._bns = []
        self._bwd_builders = []    # one per forward unit; run in REVERSE so store/accumulate modes follow run order
        self.units = []            # (kind, state_dict prefix, inputs, output) per forward unit, for per-unit parity tests
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
        desc = "%d->%d k%d s%d @%dx%dx%d" % (cin, cout, k, s, n, h, w)
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
        w16 = net._packed(conv.weight, net._w16)
        gw = net._packed(conv.weight, net._g32)
        if not reduced:  # else: the dgrad that produced dy already accumulated dbeta / dgamma in its epilogue
            B.add("bn_bwd_reduce", lambda: ops.bn_bwd_reduce(dy, ymask, z, bn.mean, bn.invstd, bn.dbeta, bn.dgamma),
                  0, _nb(dy, ymask, z))
        self.sync_bn_grads(B, bn)
        B.add("bn_bwd_apply", lambda: ops.bn_bwd_apply(dy, ymask, z, bn.mean, bn.invstd, bn.gamma, bn.app_dbeta,
                                                      bn.app_dgamma, dz, g_out, g_out_acc, self.bn_scale), 0,
              _nb(dy, ymask, z, dz, g_out))
        desc = "%d->%d k%d s%d @%dx%dx%d" % (x.shape[3], dz.shape[3], k, s, x.shape[0], x.shape[1], x.shape[2])
        B.add("conv_wgrad", lambda: ops.conv_wgrad(dz, x, gw, k, s), 2.0 * dz.numel() * x.shape[3] * k * k,
              _nb(dz, x, gw), desc)
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

    # ------------------------------------------------------------------------------------------ network
    def _build(self):
        net, n, h, w = self.net, self.n, self.h, self.w
        F = self.fwd_ops
        enc = net.encoder
        train = self.training

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
        if train:
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
        if train:
            def build_stem(B):
                d_a0 = self.gbuf(a0)
                d_c1 = self.gbuf(c1)
                dz0 = self.act(*z0.shape)
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
                B.add("conv_wgrad", lambda: ops.conv_wgrad(dz0, col, stem_gw, 1, 1), sflops, _nb(dz0, col))
                B.add("misc", lambda: ops.stem_unpack_wgrad(stem_gw, stem_g))
            self._bwd_builders.append(("stem", build_stem))

        # ---- encoder stages (torchvision BasicBlock / Bottleneck)
        x = c1
        skips = []
        for li, layer in enumerate((enc.layer1, enc.layer2, enc.layer3, enc.layer4)):
            for bi, blk in enumerate(layer):
                xin = x
                self._cur_tag = "layer%d" % (li + 1)
                x = self._res_block(x, blk)
                self.units.append(("block", "encoder.layer%d.%d" % (li + 1, bi), (xin,), x))
            skips.append(x)
        c2, c3, c4, c5 = skips

        # ---- centre + decoder (src/unet_models.py:373-403)
        pool = self.act(n, c5.shape[1] // 2, c5.shape[2] // 2, c5.shape[3])
        F.add("maxpool", lambda: ops.maxpool2_fwd(c5, pool), 0, _nb(c5, pool))
        if train:
            def build_pool(B):
                d_pool, d_c5 = self.gbuf(pool), self.gbuf(c5)
                acc = self.gmode(c5)  # dec5's skip dgrad ran first -> accumulate
                B.add("maxpool", lambda: ops.maxpool2_bwd(c5, d_pool, d_c5, acc), 0, _nb(c5, d_pool, d_c5))
            self._bwd_builders.append(("decoder", build_pool))
        center = self._decoder(pool, None, net.center, pool_input=True)
        d5 = self._decoder(center, c5, net.dec5)
        d4 = self._decoder(d5, c4, net.dec4)
        d3 = self._decoder(d4, c3, net.dec3)
        d2 = self._decoder(d3, c2, net.dec2)
        d1 = self._decoder(d2, None, net.dec1)
        self.units += [("decoder", "center", (pool,), center), ("decoder", "dec5", (center, c5), d5),
                       ("decoder", "dec4", (d5, c4), d4), ("decoder", "dec3", (d4, c3), d3),
                       ("decoder", "dec2", (d3, c2), d2), ("decoder", "dec1", (d2,), d1)]
        # dec0 = ConvRelu(32, 32)
        conv0 = net.dec0.conv
        w0_16 = net._packed(conv0.weight, net._w16)
        b0 = net._vec(conv0.bias, net._p32)
        d0 = self.act(n, h, w, conv0.out_channels)
        f0 = 2.0 * d0.numel() * d1.shape[3] * 9
        F.add("conv_fwd", lambda: ops.conv_fwd(d1, w0_16, 3, 1, bias=b0, relu=True, out=d0), f0, _nb(d1, d0))
        fw, fb = net._vec(net.final.weight, net._p32), net._vec(net.final.bias, net._p32)
        F.add("final_conv", lambda: ops.final_conv_fwd(d0, fw, fb, self.logits), 2.0 * self.logits.numel() * 32,
              _nb(d0, self.logits))
        self.named = dict(conv1=c1, conv2=c2, conv3=c3, conv4=c4, conv5=c5, center=center, dec5=d5, dec4=d4, dec3=d3,
                          dec2=d2, dec1=d1, dec0=d0)
        if train:
            def build_head(B):
                g_d0 = self.gbuf(d0)
                gfw, gfb = net._vec(net.final.weight, net._g32), net._vec(net.final.bias, net._g32)
                # final 1x1 backward also applies dec0's ReLU mask
                B.add("final_conv", lambda: ops.final_conv_bwd(d0, fw, self.dlogits, g_d0, gfw, gfb),
                      4.0 * self.logits.numel() * 32, _nb(d0, self.dlogits, g_d0))
                gb0 = net._vec(conv0.bias, net._g32)
                gw0 = net._packed(conv0.weight, net._g32)
                B.add("channel_sum", lambda: ops.channel_sum(g_d0, gb0), 0, _nb(g_d0))
                B.add("conv_wgrad", lambda: ops.conv_wgrad(g_d0, d1, gw0, 3, 1), f0, _nb(g_d0, d1))
                self.dgrad_into(B, g_d0, conv0, d1, relu_mask=d1)
            self._bwd_builders.append(("decoder", build_head))

    def _res_block(self, x, blk):
        """torchvision BasicBlock / Bottleneck forward + backward plan"""
        train = self.training
        F = self.fwd_ops
        is_bottleneck = hasattr(blk, "conv3")
        convs = [(blk.conv1, blk.bn1), (blk.conv2, blk.bn2)] + ([(blk.conv3, blk.bn3)] if is_bottleneck else [])
        if not train:
            cur = x
            for conv, bnm in convs[:-1]:
                cur, _, _ = self.conv_bn(cur, conv, bnm, True)
            ident = x
            if blk.downsample is not None:
                ident, _, _ = self.conv_bn(x, blk.downsample[0], blk.downsample[1], False)
            out, _, _ = self.conv_bn(cur, convs[-1][0], convs[-1][1], True, residual=ident)
            return out
        acts = [x]
        units = []
        cur = x
        for conv, bnm in convs[:-1]:
            y, z, bn = self.conv_bn(cur, conv, bnm, True)
            units.append((conv, cur, y, z, bn))
            cur = y
        conv_l, bn_l = convs[-1]
        _, z_l, bnl = self.conv_bn(cur, conv_l, bn_l, None)
        out = self.act(*z_l.shape)
        if blk.downsample is not None:
            dconv, dbnm = blk.downsample[0], blk.downsample[1]
            _, zd, bnd = self.conv_bn(x, dconv, dbnm, None)
            self.bn_apply_op(z_l, bnl, out, True, zd, bnd)
        else:
            self.bn_apply_op(z_l, bnl, out, True, x)
        if train:
            last_in = cur

            def build_block(B):
                d_out = self.gbuf(out)
                if blk.downsample is None:
                    # identity branch: grad(x) (+)= g = d_out * (out > 0), emitted by the last BN's backward pass
                    gx = self.gbuf(x)
                    acc = self.gmode(x)
                    dz_l = self.conv_unit_backward(B, d_out, out, z_l, bnl, conv_l, last_in, g_out=gx, g_out_acc=acc)
                else:
                    dz_l = self.conv_unit_backward(B, d_out, out, z_l, bnl, conv_l, last_in)
                # walk back through the inner units
                dz = dz_l
                conv_next = conv_l
                for conv, xin, y, z, bn in reversed(units):
                    # y has a single consumer: its ReLU mask and its BN's backward reductions ride in the dgrad epilogue
                    self.dgrad_into(B, dz, conv_next, y, bn_reduce=(z, bn))
                    dz = self.conv_unit_backward(B, self.gbuf(y), None, z, bn, conv, xin, reduced=True)
                    conv_next = conv
                self.dgrad_into(B, dz, conv_next, x)
                if blk.downsample is not None:
                    dzd = self.conv_unit_backward(B, d_out, out, zd, bnd, dconv, x)
                    self.dgrad_into(B, dzd, dconv, x)
            self._bwd_builders.append((self._cur_tag, build_block))
        return out

    def _decoder(self, x1, skip, block, pool_input=False):
        """DecoderBlockV2: relu(conv3x3(cat[x1, skip]) + b) -> relu(convT4x4s2(.) + b)   (src/unet_models.py:136-141)"""
        net = self.net
        F = self.fwd_ops
        conv, deconv = block.block[0].conv, block.block[1]
        n, h, w, c1 = x1.shape
        cmid, cout = conv.out_channels, deconv.out_channels
        w16 = net._packed(conv.weight, net._w16)
        b1 = net._vec(conv.bias, net._p32)
        wt16 = net._packed(deconv.weight, net._w16)
        b2 = net._vec(deconv.bias, net._p32)
        mid = self.act(n, h, w, cmid)
        out = self.act(n, 2 * h, 2 * w, cout)
        ctot = c1 + (skip.shape[3] if skip is not None else 0)
        if self.training:
            self.bias_sum[id(out)] = net._vec(deconv.bias, net._g32)
        fc = 2.0 * mid.numel() * ctot * 9
        ft = 2.0 * mid.numel() * cout * 16
        F.add("conv_fwd", lambda: ops.conv_fwd(x1, w16, 3, 1, bias=b1, relu=True, x2=skip, out=mid), fc,
              _nb(x1, skip, w16, mid), "dec %d->%d k3 @%dx%dx%d" % (ctot, cmid, n, h, w))
        F.add("convt_fwd", lambda: ops.convt_fwd(mid, wt16, bias=b2, relu=True, out=out), ft, _nb(mid, wt16, out),
              "%d->%d @%dx%dx%d" % (cmid, cout, n, h, w))
        if self.training:
            def build_dec(B):
                g_out = self.gbuf(out)   # already masked by out's ReLU (the consumer's dgrad epilogue did it)
                g_mid = self.gbuf(mid)
                gwt = net._packed(deconv.weight, net._g32)
                gb2 = net._vec(deconv.bias, net._g32)
                gw = net._packed(conv.weight, net._g32)
                gb1 = net._vec(conv.bias, net._g32)
                if id(out) not in self.bias_fused:   # else: summed in the epilogue of the dgrad that produced g_out
                    B.add("channel_sum", lambda: ops.channel_sum(g_out, gb2), 0, _nb(g_out))
                dd = "%d->%d @%dx%dx%d" % (cmid, cout, n, h, w)
                B.add("convt_wgrad", lambda: ops.convt_wgrad(g_out, mid, gwt), ft, _nb(g_out, mid, gwt), dd)
                B.add("convt_dgrad", lambda: ops.convt_dgrad(g_out, wt16, relu_mask=mid, out=g_mid, channel_sum=gb1), ft,
                      _nb(g_out, wt16, mid, g_mid), dd)
                B.add("conv_wgrad", lambda: ops.conv_wgrad(g_mid, x1, gw, 3, 1, ci_off=0),
                      2.0 * mid.numel() * c1 * 9, _nb(g_mid, x1), "dec %d->%d k3 @%dx%dx%d" % (c1, cmid, n, h, w))
                if skip is not None:
                    B.add("conv_wgrad", lambda: ops.conv_wgrad(g_mid, skip, gw, 3, 1, ci_off=c1),
                          2.0 * mid.numel() * skip.shape[3] * 9, _nb(g_mid, skip),
                          "dec-skip %d->%d k3 @%dx%dx%d" % (skip.shape[3], cmid, n, h, w))
                # x1 is a decoder ReLU output (mask in the epilogue) unless it is the centre's max-pool output
                self.dgrad_into(B, g_mid, conv, x1, relu_mask=None if pool_input else x1, ci_off=0)
                if skip is not None:
                    self.dgrad_into(B, g_mid, conv, skip, relu_mask=None, ci_off=c1)
            self._bwd_builders.append(("decoder", build_dec))
        return out

    # ------------------------------------------------------------------------------------------ execution
    def _bn_table(self):
        if getattr(self, "_bn_tab", None) is None:
            rows = [[b.gamma.data_ptr(), b.beta.data_ptr(), b.mod.running_mean.data_ptr(), b.mod.running_var.data_ptr(),
                     b.scale.data_ptr(), b.shift.data_ptr(), b.c] for b in self._bns]
            self._bn_tab = torch.tensor(rows, dtype=torch.int64, device=self.dev)
            self._bn_maxc = max(b.c for b in self._bns)
        return self._bn_tab

    def _run_fwd(self):
        if not self.training:
            tab = self._bn_table()
            L.fcall("mcb_bn_eval_params_batched", tab.data_ptr(), len(self._bns), self._bn_maxc, BN_EPS)
        if self.training:
            if self.sync_nvlink:
                L.fcall("mcb_sync_step_bump", self._sync_step.data_ptr())
            L.zero(self._stats_arena)
        for op in self.fwd_ops:
            op()

    def _run_bwd(self, first=0, last=None, hooks=None):
        """backward layers [first, last) in execution (reverse-forward) order; the gradient arena is zeroed with the
        first layer.  hooks = {layer_index: fn}: fn() runs ON THE SIDE STREAM once every launch of the layers before
        `layer_index` (main chain and weight-gradient GEMMs) is ordered before it -- used for per-segment optimizer
        updates that overlap the rest of the backward pass."""
        if first == 0:
            L.zero(self.net._g32)
            if self.sync_nvlink:
                L.zero(self._dstats_loc)
        # Weight/bias-gradient launches are leaves of the backward graph (they only add into the gradient arena): they
        # go to a side stream, forked after their producer and joined at the end, so the tensor-core-bound wgrad GEMMs
        # overlap the HBM-bound BatchNorm-backward kernels of the layers below instead of queueing behind them.
        # (No buffer is recycled inside a step, so the only hazards are the recorded producer -> consumer edges.)
        use_side = os.environ.get("MCB_SIDE_WGRAD", "1") == "1"
        main = torch.cuda.current_stream()
        if use_side and self._side is None:
            self._side = torch.cuda.Stream(device=self.dev)
        forked = False
        pending = []
        # with prioritised streams the side work cannot delay the main chain, so it starts as early as possible;
        # without them a weight-gradient GEMM is held back until the next data-gradient GEMM has been launched
        defer = os.environ.get("MCB_SIDE_DEFER", "0" if stream_priority_enabled() else "1") == "1"

        def flush():
            nonlocal forked
            if not pending:
                return
            ev = torch.cuda.Event()
            ev.record(main)
            self._side.wait_event(ev)
            with torch.cuda.stream(self._side):
                for q in pending:
                    q()
            pending.clear()
            forked = True

        def run_hook(idx):
            nonlocal forked
            if hooks and idx in hooks:
                if not use_side:
                    hooks[idx]()
                    return
                flush()
                ev = torch.cuda.Event()
                ev.record(main)
                self._side.wait_event(ev)
                with torch.cuda.stream(self._side):
                    hooks[idx]()
                forked = True

        n_layers = len(self.bwd_layers) if last is None else last
        for li, layer in enumerate(self.bwd_layers[first:last], start=first):
            run_hook(li)
            for op in layer:
                if use_side and op.kind in _SIDE_KINDS and op.desc:
                    pending.append(op)
                    if not defer:
                        flush()
                else:
                    op()
                    # a deferred wgrad starts right AFTER the next data-gradient GEMM (which needs whole SMs), i.e.
                    # next to the BatchNorm-backward kernels that follow it
                    if op.kind in ("conv_dgrad", "convt_dgrad"):
                        flush()
        flush()
        run_hook(n_layers)
        if forked:
            ev = torch.cuda.Event()
            ev.record(self._side)
            main.wait_event(ev)

    def bwd_segments(self):
        """split points for overlapping the gradient all-reduce / the Adam update with the backward pass:
        [decoder | layer4 | layer3 | rest].  -> [(first_layer, last_layer, arena_lo, arena_hi)], the arena range is
        complete once the segment has run (layer3's 23 blocks reduce while layer2 / layer1 / stem still run)"""
        net = self.net
        tags = self.bwd_tags
        n = len(tags)
        i_dec = max(i for i, t in enumerate(tags) if t == "decoder") + 1
        i_l4 = max(i for i, t in enumerate(tags) if t == "layer4") + 1
        i_l3 = max(i for i, t in enumerate(tags) if t == "layer3") + 1
        off = {name: net._slots[id(p)].off for name, p, _ in net._arena_params()}
        total = net._p32.numel()
        o_dec = off["center.block.0.conv.weight"]
        o_l4 = off["encoder.layer4.0.conv1.weight"]
        o_l3 = off["encoder.layer3.0.conv1.weight"]
        return [(0, i_dec, o_dec, total), (i_dec, i_l4, o_l4, o_dec), (i_l4, i_l3, o_l3, o_l4), (i_l3, n, 0, o_l3)]

    def forward(self, x, use_graph=True):
        self.x_in.copy_(x)
        if not use_graph:
            self._run_fwd()
            return self.logits
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

    def backward(self, dlogits, use_graph=True):
        self.dlogits.copy_(dlogits)
        if not use_graph:
            self._run_bwd()
            return
        if self.graph_bwd is None:
            self._run_bwd()
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with graph_capture(g, self.dev):
                self._run_bwd()
            self.graph_bwd = g
            return
        self.graph_bwd.replay()


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
