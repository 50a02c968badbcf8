"""TEST INFRASTRUCTURE -- the harness of the convolution-kernel tests, each of which covers one regime:
tests/test_conv_gemm_gpu.py (small shapes, about one tile per CTA), tests/test_conv_gemm_persistent_gpu.py (several
tiles per CTA, every test hook), tests/test_conv_gemm_epilogue_overlap_gpu.py (the hand-off to the epilogue warpgroup),
tests/test_conv_gemm_encoders_gpu.py (the 3x3 transposed conv) and tests/test_vgg_kernels_gpu.py (the VGG input and
concat convs).  tests/test_elementwise_gpu.py takes its layout helpers.  Never imported by the product path; mcb200 is
imported inside the functions, once the mcb fixture has built it.

A case is a dict: desc (the seed key), n, h, w, cout, k, s (stride, 1 if absent), and the input channels of the conv:
c0 and c1 (a concatenated second source, 0 if absent) for the forward references, cin for the others.

References are float64 on the CPU from the bf16-rounded operands.  Each comes with A, the same operation on |operands|,
which scales the fp32 accumulation error.  The bar, assert_bound, element-wise:
  bf16 outputs   |got - ref| <= 2^-8 |ref| + 2^-16 A: half a bf16 ulp plus an accumulation allowance far above the
                 realistic ~2^-24 A and far below one dropped product term, tap or channel chunk;
  fp32 results   |got - ref| <= 2^-16 A (rel = 0): weight gradients, and the fused per-channel sums against the float64
                 sum of the STORED output (check_sums);
  integer-exact  bitwise (assert_exact): operands in {-1, 0, 1}, |ref| <= 256, sums < 2^24.
Real-valued fused reductions must also repeat bitwise from run to run (assert_same)."""
import itertools
import zlib

import pytest
import torch
import torch.nn.functional as F


# ----------------------------------------------------------------------------------------------- layout and rounding
def nhwc(x):
    return x.permute(0, 2, 3, 1).contiguous()


def nchw(x):
    return x.permute(0, 3, 1, 2).contiguous()


def bf16r(x):
    """x rounded to bf16, as float32 (exact, as is its .double())"""
    return x.to(torch.bfloat16).float()


def dev(x):
    """NCHW float -> NHWC bf16 on the GPU"""
    return nhwc(x).to("cuda", torch.bfloat16)


def pack(wt):
    """conv weight (cout, cin, k, k) -> bf16 (taps, cout, cin) on the GPU"""
    from mcb200 import ops
    return ops.pack_conv_weight(wt).to("cuda", torch.bfloat16)


def pack_t(wt):
    """transposed-conv weight (cin, cout, k, k) -> bf16 (taps, cout, cin) on the GPU"""
    from mcb200 import ops
    return ops.pack_convt_weight(wt).to("cuda", torch.bfloat16)


# -------------------------------------------------------------------------------------------------- seeded operands
def gen(*key):
    return torch.Generator().manual_seed(zlib.crc32(repr(key).encode()))


def ints(g, shape, density=1.0):
    """values in {-1, 0, 1}; a nonzero with probability 2/3 * density"""
    v = torch.randint(-1, 2, shape, generator=g).float()
    return v * (torch.rand(shape, generator=g) < density).float() if density < 1 else v


def int_density(k_terms):
    """weight density for K-term integer dot products: E[v^2] = 16, so max|v| stays far below 256 and the per-channel
    sums of v^2 over <= 10^5 pixels below 2^24"""
    return min(1.0, 24.0 / k_terms)


def cached(cache, key, make):
    """make(gen(*key)), kept under key in cache, the calling test module's dict (None: not kept)"""
    if cache is None:
        return make(gen(*key))
    if key not in cache:
        cache[key] = make(gen(*key))
    return cache[key]


def sweep(cases, *axes, halo=False):
    """pytest params: case x its BN list x (halo: its MCB_HALO list, the default rule if it has none) x axes"""
    out = []
    for c in cases:
        for bn in c.get("bn", (None,)):
            for hm in c.get("halo", (2,)) if halo else (None,):
                for vs in itertools.product(*axes):
                    args = [c] + [a for a in (bn, hm) if a is not None] + list(vs)
                    parts = [c["desc"].replace(" ", "_")] + (["BN%d" % bn] if bn else []) + \
                        (["halo%d" % hm] if halo and "halo" in c else []) + list(vs)
                    out.append(pytest.param(*args, id="-".join(parts)))
    return out


# --------------------------------------------------------------------------------------------------------- the bar
def assert_bound(got, ref, absref, what, rel=2.0 ** -8, extra=0.0):
    """|got - ref| <= rel |ref| + 2^-16 absref + extra element-wise (rel = 0, absref = 0: exact), on got's device"""
    got = got.double()
    d = got.device
    ref = ref.to(d, torch.float64)
    absref = absref.to(d, torch.float64) if torch.is_tensor(absref) else absref
    extra = extra.to(d, torch.float64) if torch.is_tensor(extra) else extra
    err = (got - ref).abs()
    bad = ~(err <= rel * ref.abs() + 2.0 ** -16 * absref + extra)  # (NaN counts as bad)
    if bad.any():
        i = tuple(int(v) for v in bad.nonzero()[0])
        a = float(absref[i]) if torch.is_tensor(absref) else absref
        raise AssertionError("%s: %d/%d elements off, max err %g; first at %s: got %r, ref %r, A %g" % (
            what, int(bad.sum()), bad.numel(), float(err.nan_to_num(float("inf")).max()), i, float(got[i]),
            float(ref[i]), a))


def assert_exact(got, ref, what):
    assert_bound(got, ref, 0.0, what, rel=0.0)


def assert_same(a, b, what):
    """bitwise repeat of a run"""
    assert torch.equal(a, b), "%s: two runs differ in %d elements" % (what, int((a != b).sum()))


def assert_accumulated(got, pre, ref, absref, what):
    """got = bf16(pre + bf16(acc)): two roundings, so the bar on pre + ref gains the first one's 2^-8 |ref|, and the
    2^-8 of that which the second one adds.  Where ref and A are zero (pixels the kernel must not touch) this demands
    got == pre."""
    assert_bound(got, pre.double() + ref, absref, what, extra=(2.0 ** -8 + 2.0 ** -16) * ref.abs())


def check_sums(got, stored, what, exact):
    """a fused per-channel sum against the float64 sum of what the kernel stored (stored: N, C, H, W)"""
    stored = stored.double()
    s, a = stored.sum((0, 2, 3)), stored.abs().sum((0, 2, 3))
    if exact:
        assert a.max() < 2 ** 24
        assert_exact(got, s, what)
    else:
        assert_bound(got, s, a, what, rel=0.0)


# ------------------------------------------------------------------------------------------------ float64 references
def fwd_ref(c, exact, cache=None):
    """forward conv: x (the sources side by side), wt, b, then conv(x, wt) and conv(|x|, |wt|), both without bias"""
    def make(g):
        cin, k, cout = c["c0"] + c.get("c1", 0), c["k"], c["cout"]
        if exact:
            x = ints(g, (c["n"], cin, c["h"], c["w"]))
            wt = ints(g, (cout, cin, k, k), int_density(cin * k * k))
            b = torch.randint(-3, 4, (cout,), generator=g).float()
        else:
            x = bf16r(torch.randn(c["n"], cin, c["h"], c["w"], generator=g))
            wt = bf16r(torch.randn(cout, cin, k, k, generator=g) / (cin * k * k) ** 0.5)
            b = torch.randn(cout, generator=g)
        conv = lambda a, v: F.conv2d(a.double(), v.double(), stride=c.get("s", 1), padding=k // 2)
        return x, wt, b, conv(x, wt), conv(x.abs(), wt.abs())
    return cached(cache, ("fwd", c["desc"], exact), make)


def run_fwd(c, x, wt, **kw):
    """conv_fwd of case c on the GPU, the second source (if any) as x2"""
    from mcb200 import ops
    c0 = c["c0"]
    x2 = dev(x[:, c0:]) if c.get("c1") else None
    return ops.conv_fwd(dev(x[:, :c0]), pack(wt), c["k"], c.get("s", 1), x2=x2, **kw)


def bn_operands(g, shape, exact):
    """z, mean, invstd, gamma, beta of a producing conv-BN-ReLU unit; exact: power-of-two scales and integer shifts, so
    the mask, xhat and both sums are exact"""
    ch = shape[1]
    if exact:
        z = torch.randint(-3, 4, shape, generator=g).float()
        mean = torch.randint(-1, 2, (ch,), generator=g).float()
        invstd = 2.0 ** torch.randint(-1, 2, (ch,), generator=g).float()
        gamma = 2.0 ** torch.randint(-1, 2, (ch,), generator=g).float() * \
            (2 * torch.randint(0, 2, (ch,), generator=g) - 1)
        beta = torch.randint(-1, 2, (ch,), generator=g).float()
    else:
        z = bf16r(torch.randn(shape, generator=g) * 1.5 + 0.3)
        mean, invstd = torch.randn(ch, generator=g) * 0.2, torch.rand(ch, generator=g) + 0.5
        gamma, beta = torch.randn(ch, generator=g), torch.randn(ch, generator=g) * 0.5
    return z, mean, invstd, gamma, beta


def bn_terms(bnp):
    """the producing unit's BatchNorm output (its sign is the ReLU mask) and xhat, float64"""
    z, mean, invstd, gamma, beta = bnp
    v = lambda t: t.double().view(1, -1, 1, 1)
    sc = gamma * invstd
    return z.double() * v(sc) + v(beta - mean * sc), (z.double() - v(mean)) * v(invstd)


def bn_reduce(bnp):
    """conv_dgrad's bn_reduce operands on the GPU: z, mean, invstd, gamma, beta, then dbeta and dgamma, zeroed"""
    z, *vecs = bnp
    return (dev(z),) + tuple(v.to("cuda") for v in vecs) + (torch.zeros(z.shape[1], device="cuda"),
                                                             torch.zeros(z.shape[1], device="cuda"))


def dgrad_ref(c, exact, cache=None):
    """data gradient of the conv cin -> cout: dy, wt, act (the producing layer's ReLU output, for relu_mask), the
    producing unit's BatchNorm operands (for bn_reduce), then dx and A"""
    def make(g):
        n, h, w, cin, cout, k, s = c["n"], c["h"], c["w"], c["cin"], c["cout"], c["k"], c.get("s", 1)
        if exact:
            dy = ints(g, (n, cout, h // s, w // s))
            wt = ints(g, (cout, cin, k, k), int_density(cout * k * k))
        else:
            dy = bf16r(torch.randn(n, cout, h // s, w // s, generator=g))
            wt = bf16r(torch.randn(cout, cin, k, k, generator=g) / (cout * k * k) ** 0.5)
        act = bf16r(torch.randn(n, cin, h, w, generator=g))
        bnp = bn_operands(gen("bnred", c["desc"], exact), (n, cin, h, w), exact)
        dg = lambda v, d: torch.nn.grad.conv2d_input((n, cin, h, w), v.double(), d.double(), stride=s,
                                                     padding=k // 2)
        return dy, wt, act, bnp, dg(wt, dy), dg(wt.abs(), dy.abs())
    return cached(cache, ("dgrad", c["desc"], exact), make)


def wgrad_ref(c, exact, cache=None):
    """weight gradient of the conv cin -> cout: x, dy, then dW and A as (cout, cin, k, k)"""
    def make(g):
        n, h, w, cin, cout, k, s = c["n"], c["h"], c["w"], c["cin"], c["cout"], c["k"], c.get("s", 1)
        if exact:
            x, dy = ints(g, (n, cin, h, w)), ints(g, (n, cout, h // s, w // s))
        else:
            x = bf16r(torch.randn(n, cin, h, w, generator=g))
            dy = bf16r(torch.randn(n, cout, h // s, w // s, generator=g))
        wg = lambda a, d: torch.nn.grad.conv2d_weight(a.double(), (cout, cin, k, k), d.double(), stride=s,
                                                      padding=k // 2)
        return x, dy, wg(x, dy), wg(x.abs(), dy.abs())
    return cached(cache, ("wgrad", c["desc"], exact), make)


def convt_ref(c, exact, cache=None):
    """transposed conv cin -> cout, stride 2, padding 1, k 4 (the default) or 3 with output_padding 1: operands x, wt,
    dy, b, act (the ReLU output of x's producer), then y (without bias), dx, dW (cin, cout, k, k), then the same on
    |operands|"""
    def make(g):
        n, h, w, cin, cout, k = c["n"], c["h"], c["w"], c["cin"], c["cout"], c.get("k", 4)
        if exact:
            x = ints(g, (n, cin, h, w))
            wt = ints(g, (cin, cout, k, k), int_density(k * k * cout))  # about k^2 / 4 cin terms forward, k^2 cout back
            dy = ints(g, (n, cout, 2 * h, 2 * w))
            b = torch.randint(-3, 4, (cout,), generator=g).float()
        else:
            x = bf16r(torch.randn(n, cin, h, w, generator=g))
            wt = bf16r(torch.randn(cin, cout, k, k, generator=g) / (cin * k * k / 4) ** 0.5)
            dy = bf16r(torch.randn(n, cout, 2 * h, 2 * w, generator=g))
            b = torch.randn(cout, generator=g)
        act = bf16r(torch.randn(n, cin, h, w, generator=g))

        def grads(xv, wv, dv):
            xr, wr = xv.double().requires_grad_(True), wv.double().requires_grad_(True)
            y = F.conv_transpose2d(xr, wr, stride=2, padding=1, output_padding=k % 2)
            y.backward(dv.double())
            return y.detach(), xr.grad, wr.grad
        return (x, wt, dy, b, act) + grads(x, wt, dy) + grads(x.abs(), wt.abs(), dy.abs())
    return cached(cache, ("convt", c["desc"], exact), make)


# ------------------------------------------------------------------------------------------------------ tile model
def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def pick_tile(wv, hv, n, max_rows, row_mult):
    """the pixel tile count of the host's box choice, a copy of its rule (csrc/conv_gemm.cu: pick_tile).  The conv GEMMs
    call it with max_rows 128, row_mult 1 (unless the haloed 8x16 box is taken), the weight gradients with 64, 16."""
    best, choice = -1.0, (1, 1, 1)
    for bw in range(1, min(max_rows, wv, 256) + 1):
        bh = 1
        while bw * bh <= max_rows and bh <= min(hv, 256):
            for bn in range(1, min(256, max_rows // (bw * bh)) + 1):
                if bn > n and row_mult == 1:
                    break
                if (bw * bh * bn) % row_mult:
                    continue
                tiles = -(-wv // bw) * -(-hv // bh) * -(-n // bn)
                score = wv * hv * n / (tiles * max_rows) + 1e-6 * bw + 1e-9 * bh
                if score > best:
                    best, choice = score, (bw, bh, bn)
            bh += 1
    bw, bh, bn = choice
    return -(-wv // bw) * -(-hv // bh) * -(-n // bn)


def tile_count(n, hv, wv, n_extent, bn, phases=1, any_box=False):
    """tiles of one conv GEMM launch over n images of hv x wv output pixels (per phase) and n_extent output channels, in
    N tiles of bn, the width forced through MCB_FORCE_BN.  The host ignores a forced bn that does not divide n_extent;
    for such a bn, and for None (the default rule), the count takes one N tile, a lower bound.  any_box: the pixel tiles
    as a lower bound that holds for whichever box the host picks, the haloed one included, as no box has more than 128
    rows; otherwise the exact count of the unhaloed box."""
    bn = bn if bn and n_extent % bn == 0 else n_extent
    pixel_tiles = -(-n * hv * wv // 128) if any_box else pick_tile(wv, hv, n, 128, 1)
    return pixel_tiles * (n_extent // bn) * phases


def assert_tiles_per_cta(count, at_least):
    """every CTA of the persistent grid (min(tiles, SMs) CTAs) runs at least at_least tiles"""
    assert count >= at_least * sms(), "only %d tiles for %d SMs, want %d per CTA" % (count, sms(), at_least)


# ------------------------------------------------------------------------------------------------------- test hooks
def set_knobs(monkeypatch, bn=None, halo=None, splits=None):
    """MCB_FORCE_BN, MCB_HALO (0 never, 1 wherever the haloed tile fits, 2 the default rule), MCB_WGRAD_SPLITS; each
    one not given is unset"""
    for name, v in (("MCB_FORCE_BN", bn), ("MCB_HALO", halo), ("MCB_WGRAD_SPLITS", splits)):
        if v is None:
            monkeypatch.delenv(name, raising=False)
        else:
            monkeypatch.setenv(name, str(v))
