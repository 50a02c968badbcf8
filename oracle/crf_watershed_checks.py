"""TEST INFRASTRUCTURE -- the harness of the dense-CRF and watershed tests (csrc/crf.cu, csrc/watershed.cu):
tests/test_crf_watershed_cpu.py and tests/test_crf_watershed_scale_gpu.py.  Never imported by the product path.

Dense CRF.  crf_f64 restates oracle/post_oracle.py::dense_crf in float64 with torch (plain shifts and adds, none of this
project's kernels), so it runs on the device at the inference batch size or on the CPU.  The parameters enter rounded to
float32, as the library receives them.  Bars:

  * one step (crf_one_step, the main check).  The device output Q_k for `iterations = k` must equal ONE float64 step
    taken from the device's own Q_(k-1) (from the clipped probabilities when k = 1).  Mean-field amplifies earlier
    errors by up to (|compat_g| + |compat_b|) / 2 per iteration, so comparing k iterations end to end says little about
    the kernel; one step from the kernel's own state measures the error of that step alone.  The bar is a running error
    bound, evaluated per pixel alongside the reference (u = 2^-24, the fp32 unit roundoff):
      - bilateral tap j of pixel i: the weight 2^-t comes from ex2.approx.ftz.f32 (2 ulp = 2^-22 relative: CUDA C
        Programming Guide, exp2f, which compiles to it) of a t rounded in fp32.  t = e1b[dx] + |s dI|^2 (s = fp32
        colour scale) carries |dt| <= u (8 t + s^2 (1020 sum|dI| + 3)): three fma roundings and e1b's rounding (4 u t),
        and the colour differences of pre-scaled fp32 colours (up to 255 s each, so cancellation costs 1020 s^2 |dI|
        absolute).  So tap j is off by 2^-22 + u (vertical weight) + ln 2 |dt| relative; ftz flushes below 2^-126;
      - the 169-tap sum: 13 taps per row, then 13 rows through fma with the vertical weight: 26 u of its magnitude
        (every term is >= 0, so the magnitude is the message itself); q n_b costs u, the final scaling u;
      - the separable Gaussian message, 13 + 13 taps: 2 u for the fp32 weights, u for q n_g, 26 u of depth, its norm
        16 u (sum 28 u, sqrtf and the reciprocal 2 u) at both ends, and the final scaling: 62 u of the message;
      - the norms n = 1 / sqrt(sum K + 1e-20): half the sum's relative error plus 2 u;
      - the energy E_c = logf(p_c) + cg msg_g + cb msg_b: logf 2 u |log p| (1 ulp), four roundings of the magnitude;
      - the softmax: expf (2 ulp), the argument's rounding, the sum and the division: 12 u absolute;
      - a two-class softmax has slope at most 1/4 in E_1 - E_0: |dQ| <= (dE_0 + dE_1) / 4 + 12 u;
      - at k = 1 the kernel's own Q_0 (logf, expf, division in fp32) is off by eta = (2 u |log p_0| + 2 u |log p_1|) / 4
        + 12 u, which enters the messages through their (non-negative) weights.
    The same bound with the fp32 numpy oracle's error model (ORACLE_F32) pins crf_f64 against post_oracle.dense_crf.
  * end to end: E2E_BAR = 1e-4 max-abs after 5 iterations, the CRF bar of the existing tests.
  * truncation: the crf.cu header claims that at the refusal bound sxy = SXY_MAX the 13x13 window stays within
    TRUNCATION_BAR of a full-window filter (5 iterations, default compatibilities, noise images).

Watershed.  watershed_ref_batched restates the three relaxations of post_oracle.minimax_watershed in int64 torch,
vectorised over planes, and is equal to it bit for bit; the kernel must be equal to both bit for bit.

Generators: a serpentine corridor, a square spiral inside one 32x32 tile, plateaus with several markers and dark-bordered
RGB images (near-black pixels at the image edge are where staging an off-image pixel with a real colour would show)."""
import math

import numpy as np
import torch
import torch.nn.functional as F

from oracle import post_oracle as P

U = 2.0 ** -24
LN2 = math.log(2.0)
EX2_REL = 2.0 ** -22                            # ex2.approx.ftz.f32: 2 ulp
CLIP = float(np.float32(1e-5))                  # the 1e-5 clip of unary_from_softmax, in fp32
SXY_MAX = 7.0 / math.sqrt(2.0 * math.log(1e7))  # crf.cu refuses wider kernels: 1.2329...
E2E_BAR = 1e-4
TRUNCATION_BAR = 4e-5
DEFAULTS = dict(compat_gaussian=3.0, sxy_gaussian=1.0, compat_bilateral=10.0, sxy_bilateral=1.0, srgb=50.0)

# per-term error models of the bound (see the module docstring): bilateral weight w_a + u (w_b x + w_c (1020 sum|dI| +
# 3) / (2 srgb^2)) relative, x = the natural exponent; Gaussian weight g_rel; sum depths in u
KERNEL = dict(w_a=EX2_REL + U, w_b=8.01, w_c=1.001, g_rel=2 * U, depth_b=26, depth_g=26, log_rel=2 * U)
# post_oracle.dense_crf: two float32 exps (numpy's SIMD exp is within 4 u) of arguments rounded twice, the products
# with the mask and with q rounded; every sum runs over all taps in sequence
ORACLE_F32 = dict(w_a=11 * U, w_b=2.0, w_c=0.0, g_rel=3 * U, depth_b=169, depth_g=169, log_rel=4 * U)


def f32(x):
    return float(np.float32(x))


def sxy_accepted(s):
    """crf.cu's refusal test on the fp32 width it receives: the heaviest dropped tap exp(-7^2 / (2 sxy^2)) <= 1e-7"""
    s = f32(s)
    return math.exp(-0.5 * 49.0 / (s * s)) <= 1e-7


def _widest_sxy():
    s = np.float32(SXY_MAX)
    while not sxy_accepted(s):
        s = np.nextafter(s, np.float32(0))
    while sxy_accepted(np.nextafter(s, np.float32(2))):
        s = np.nextafter(s, np.float32(2))
    return float(s)


SXY_OK = _widest_sxy()   # the widest fp32 sxy the library accepts, 1.2328951 (fp32 1.2329 is just above the bound)


def crf_params(**kw):
    """the CRF parameters as the library receives them (fp32)"""
    p = dict(DEFAULTS, **kw)
    return {k: f32(v) for k, v in p.items()}


def crf_rgb_ref(imgs):
    """post_oracle.crf_rgb_image for a batch: (N,3,H,W) float -> (N,H,W,3) uint8 (float64, truncate, wrap modulo 256)"""
    x = imgs.to(torch.float64)
    mean = torch.tensor(P.MEAN, dtype=torch.float64, device=x.device).view(1, 3, 1, 1)
    std = torch.tensor(P.STD, dtype=torch.float64, device=x.device).view(1, 3, 1, 1)
    v = ((x * std + mean) * 255.0).to(torch.int64) & 255
    return v.to(torch.uint8).permute(0, 2, 3, 1).contiguous()


class _Field:
    """one batch of images, padded by `radius`: tap(dy, dx) gives the in-image indicator, both kernels' weights and the
    bilateral weights' relative error bound for the shift (dy, dx)"""

    def __init__(self, rgb, params, radius, model=None):
        self.r, self.p, self.model = radius, params, model
        self.n, self.h, self.w = rgb.shape[:3]
        self.dev = rgb.device
        self.rgb = rgb.permute(0, 3, 1, 2).to(torch.float64)
        self.rgb_p = self.pad(self.rgb)
        self.in_p = self.pad(torch.ones((self.n, 1, self.h, self.w), dtype=torch.float64, device=self.dev))

    def pad(self, a):
        return F.pad(a, (self.r,) * 4)

    def sh(self, a, dy, dx):
        """a[y + dy, x + dx] of a padded array"""
        r = self.r
        return a[:, :, r + dy:r + dy + self.h, r + dx:r + dx + self.w]

    def taps(self):
        return [(dy, dx) for dy in range(-self.r, self.r + 1) for dx in range(-self.r, self.r + 1)]

    def tap(self, dy, dx):
        p = self.p
        d2 = float(dy * dy + dx * dx)
        m = self.sh(self.in_p, dy, dx)
        di = self.rgb - self.sh(self.rgb_p, dy, dx)
        x = 0.5 * d2 / p["sxy_bilateral"] ** 2 + 0.5 * (di * di).sum(1, keepdim=True) / p["srgb"] ** 2
        kg = math.exp(-0.5 * d2 / p["sxy_gaussian"] ** 2) * m
        kb = torch.exp(-x) * m
        if self.model is None:
            return kg, kb, None
        mo = self.model
        cterm = (1020.0 * di.abs().sum(1, keepdim=True) + 3.0) / (2.0 * p["srgb"] ** 2)
        rel = mo["w_a"] + U * (mo["w_b"] * x + mo["w_c"] * cterm)
        return kg, kb, rel


def _norms(fd):
    sg = torch.zeros((fd.n, 1, fd.h, fd.w), dtype=torch.float64, device=fd.dev)
    sb, eb = torch.zeros_like(sg), torch.zeros_like(sg)
    for dy, dx in fd.taps():
        kg, kb, rel = fd.tap(dy, dx)
        sg += kg
        sb += kb
        if rel is not None:
            eb += kb * rel
    ng, nb = 1.0 / torch.sqrt(sg + 1e-20), 1.0 / torch.sqrt(sb + 1e-20)
    if fd.model is None:
        return ng, nb, None, None
    mo = fd.model
    rel_ng = 0.5 * (mo["g_rel"] + mo["depth_g"] * U) + 2 * U
    rel_nb = 0.5 * (eb / sb + mo["depth_b"] * U + 169 * 2.0 ** -126) + 2 * U   # sum K >= 1: ftz as relative
    return ng, nb, rel_ng, rel_nb


def _logp(probs):
    return torch.log(torch.clamp(probs.to(torch.float64), min=CLIP))


def _step(fd, logp, q, ng, nb, rel_ng=None, rel_nb=None, eta=None):
    """one mean-field update from q -> (q_new, bar or None)"""
    p = fd.p
    qg, qb = fd.pad(q * ng), fd.pad(q * nb)
    mg, mb = torch.zeros_like(q), torch.zeros_like(q)
    bound = fd.model is not None
    if bound:
        eb = torch.zeros_like(q)                                   # sum of |term| x its relative error
        rq = fd.pad(q * nb * (rel_nb + U))                         # n_b(j) and the rounding of q n_b
        if eta is not None:
            eg_eta, eb_eta = torch.zeros_like(q), torch.zeros_like(q)
            etag, etab = fd.pad((eta * ng).expand_as(q)), fd.pad((eta * nb).expand_as(q))
    for dy, dx in fd.taps():
        kg, kb, rel = fd.tap(dy, dx)
        mg += kg * fd.sh(qg, dy, dx)
        mb += kb * fd.sh(qb, dy, dx)
        if bound:
            eb += kb * (rel * fd.sh(qb, dy, dx) + fd.sh(rq, dy, dx))
            if eta is not None:
                eg_eta += kg * fd.sh(etag, dy, dx)
                eb_eta += kb * fd.sh(etab, dy, dx)
    msg_g, msg_b = mg * ng, mb * nb
    cg, cb = p["compat_gaussian"], p["compat_bilateral"]
    e = logp + cg * msg_g + cb * msg_b
    q_new = torch.softmax(e, dim=1)
    if not bound:
        return q_new, None
    mo = fd.model
    err_g = msg_g * (mo["g_rel"] + U + 2 * rel_ng + (mo["depth_g"] + 1) * U)
    err_b = eb * nb + msg_b * (rel_nb + (mo["depth_b"] + 1) * U) + 169 * 2.0 ** -126
    if eta is not None:
        err_g = err_g + eg_eta * ng * (1 + 1e-3)
        err_b = err_b + eb_eta * nb * (1 + 1e-3)
    mag = logp.abs() + abs(cg) * msg_g + abs(cb) * msg_b
    de = mo["log_rel"] * logp.abs() + 4 * U * mag + abs(cg) * err_g + abs(cb) * err_b
    bar = 0.25 * de.sum(1, keepdim=True) + 12 * U
    return q_new, bar.expand_as(q_new)


def crf_f64(rgb, probs, params, iterations, radius=6, q0=None):
    """post_oracle.dense_crf in float64: rgb (N,H,W,3) uint8, probs (N,2,H,W), params as crf_params gives them ->
    (N,2,H,W) float64 after `iterations` mean-field updates, starting from softmax(-U) or from q0"""
    fd = _Field(rgb, params, radius)
    logp = _logp(probs)
    ng, nb, _, _ = _norms(fd)
    q = torch.softmax(logp, dim=1) if q0 is None else q0.to(torch.float64)
    for _ in range(iterations):
        q, _ = _step(fd, logp, q, ng, nb)
    return q


def crf_one_step(rgb, probs, params, q_prev=None, model=KERNEL):
    """one float64 update from q_prev (from the clipped probabilities when None) and its bar under `model` ->
    (q_ref, bar), both (N,2,H,W) float64"""
    fd = _Field(rgb, params, 6, model)
    logp = _logp(probs)
    ng, nb, rel_ng, rel_nb = _norms(fd)
    eta = None
    if q_prev is None:
        q = torch.softmax(logp, dim=1)
        eta = 0.25 * model["log_rel"] * logp.abs().sum(1, keepdim=True) + 12 * U
    else:
        q = q_prev.to(torch.float64)
    return _step(fd, logp, q, ng, nb, rel_ng, rel_nb, eta)


def normalised_from_rgb(rgb):
    """(N,H,W,3) integer colours -> (N,3,H,W) float32 ImageNet-normalised images whose crf_rgb conversion gives them
    back (the half-unit offset keeps the truncation away from the integer)"""
    x = torch.as_tensor(rgb, dtype=torch.float64).permute(0, 3, 1, 2)
    mean = torch.tensor(P.MEAN, dtype=torch.float64).view(1, 3, 1, 1)
    std = torch.tensor(P.STD, dtype=torch.float64).view(1, 3, 1, 1)
    return (((x + 0.5) / 255.0 - mean) / std).to(torch.float32).contiguous()


def dark_border_images(n, h, w, seed, border=4):
    """(N,H,W,3) uint8: random colours inside, near-black (0..3) within `border` pixels of the edge, plus a bright
    square so that the bilateral kernel sees edges"""
    rs = np.random.RandomState(seed)
    rgb = rs.randint(0, 256, (n, h, w, 3))
    edge = np.zeros((h, w), bool)
    edge[:border], edge[-border:], edge[:, :border], edge[:, -border:] = True, True, True, True
    rgb[:, edge] = rs.randint(0, 4, (n, int(edge.sum()), 3))
    rgb[:, h // 4:h // 2, w // 4:w // 2] = 240
    return rgb.astype(np.uint8)


def soft_probs(n, h, w, seed, lo=0.02, hi=0.98):
    """(N,2,H,W) float32 building probabilities with smooth structure and noise, channels summing to one"""
    rs = np.random.RandomState(seed)
    from scipy import ndimage as ndi
    p1 = np.stack([ndi.gaussian_filter(rs.randn(h, w), 2.0) for _ in range(n)])
    p1 = 1.0 / (1.0 + np.exp(-4.0 * p1 / (p1.std() + 1e-12)))
    p1 = np.clip(p1 + 0.1 * rs.randn(n, h, w), lo, hi).astype(np.float32)
    return np.stack([1 - p1, p1], axis=1).astype(np.float32)


# --------------------------------------------------------------------------------------------------------- watershed
INF = 1 << 40


def watershed_levels(prob, levels):
    """minimax_watershed's quantised relief on the planes' device: floor((1 - prob) (levels - 1)) clipped in float64
    to [0, levels - 1]; NaN goes to 0 (as prob = 1), +Inf to 0, -Inf to levels - 1"""
    v = torch.floor((1.0 - prob.to(torch.float64)) * float(levels - 1))
    v = torch.where(torch.isnan(v), torch.zeros_like(v), v.clamp(0.0, float(levels - 1)))
    return v.to(torch.int64)


def _nbrs(a):
    p = torch.full((a.shape[0], a.shape[1] + 2, a.shape[2] + 2), INF, dtype=torch.int64, device=a.device)
    p[:, 1:-1, 1:-1] = a
    return [p[:, :-2, 1:-1], p[:, 2:, 1:-1], p[:, 1:-1, :-2], p[:, 1:-1, 2:]]


def _relax(x, update, check=32):
    """apply update until a fixed point; the updates only lower values, so `check` steps without a change is one"""
    while True:
        old = x
        for _ in range(check):
            x = update(x)
        if torch.equal(x, old):
            return x


def watershed_ref_batched(prob, markers, mask, levels=256):
    """post_oracle.minimax_watershed on every plane of prob (P,H,W) float, markers (P,H,W) int, mask (P,H,W) bool, all
    torch tensors on one device -> (P,H,W) int32 labels"""
    lev = watershed_levels(prob, levels)
    mk = markers.to(torch.int64)
    is_m = mk > 0
    act = (mask.to(torch.bool) | is_m) & ~is_m
    cost = torch.where(is_m, 0, INF)

    def s1(c):
        a, b, l, r = _nbrs(c)
        cand = torch.minimum(torch.minimum(a, b), torch.minimum(l, r))
        return torch.where(act, torch.minimum(c, torch.maximum(cand, lev)), c)

    cost = _relax(cost, s1)
    ncost = _nbrs(cost)
    tight = [(torch.maximum(cq, lev) == cost) & (cq < INF) for cq in ncost]
    act2 = act & (cost < INF)

    def s2(d):
        best = torch.full_like(d, INF)
        for t, dq in zip(tight, _nbrs(d)):
            best = torch.minimum(best, torch.where(t, dq + 1, INF))
        return torch.where(act2, torch.minimum(d, best), d)

    dist = _relax(torch.where(is_m, 0, INF), s2)
    ok = [t & (dq + 1 == dist) for t, dq in zip(tight, _nbrs(dist))]
    act3 = act & (dist < INF)

    def s3(lab):
        best = torch.full_like(lab, INF)
        for o, lq in zip(ok, _nbrs(lab)):
            best = torch.minimum(best, torch.where(o, lq, INF))
        return torch.where(act3, torch.minimum(lab, best), lab)

    lab = _relax(torch.where(is_m, mk, INF), s3)
    return torch.where(lab < INF, lab, 0).to(torch.int32)


def serpentine(h, w, period=2):
    """a 1-pixel corridor snaking along rows 1, 1 + period, ... joined alternately at the right and left ends ->
    (mask (H,W) bool, order (H,W) int64: the step index along the corridor, -1 off it)"""
    order = np.full((h, w), -1, np.int64)
    k = 0
    rows = list(range(1, h - 1, period))
    for j, y in enumerate(rows):
        xs = range(1, w - 1) if j % 2 == 0 else range(w - 2, 0, -1)
        for x in xs:
            order[y, x] = k
            k += 1
        if j + 1 < len(rows):
            x = w - 2 if j % 2 == 0 else 1
            for yy in range(y + 1, rows[j + 1]):
                order[yy, x] = k
                k += 1
    return order >= 0, order


def spiral(size=32):
    """a square spiral corridor, 1 pixel wide with 1-pixel walls, filling a size x size tile from its top-left corner
    inwards -> (mask, order) as serpentine; a 32x32 spiral is 500+ steps long"""
    order = np.full((size, size), -1, np.int64)
    y, x, k = 0, 0, 0
    order[0, 0] = 0
    dirs = [(0, 1), (1, 0), (0, -1), (-1, 0)]
    lengths = [size - 1, size - 1, size - 1]
    n = size - 3
    while n > 0:
        lengths += [n, n]
        n -= 2
    for i, ln in enumerate(lengths):
        dy, dx = dirs[i % 4]
        for _ in range(ln):
            y, x, k = y + dy, x + dx, k + 1
            order[y, x] = k
    return order >= 0, order


def plateau_with_markers(h, w, points, value=0.9):
    """a flat mask of probability `value` with markers {(y, x): label}: every tie is decided by distance, then label"""
    prob = np.full((h, w), value, np.float32)
    markers = np.zeros((h, w), np.int32)
    for (y, x), lab in points.items():
        markers[y, x] = lab
    return prob, markers, np.ones((h, w), bool)


def blob_map(rs, h, w, sigma):
    from scipy import ndimage as ndi
    z = ndi.gaussian_filter(rs.randn(h, w), sigma)
    return ((z - z.min()) / (z.max() - z.min())).astype(np.float32)
