"""The inference post-processing (bench.py --workload infer) at the benchmark's batch-64 300x300 size, and the branches
of the CRF, watershed, labelling, score and morphology kernels that smaller tests never reach.

Every stage is checked on the CUDA path's own input to that stage, so an error cannot hide behind, or compound through,
an earlier one:
  * dense CRF: a float64 torch restatement of oracle/post_oracle.py::dense_crf with a `radius` parameter (the numpy
    oracle takes ~1.5 s per 300^2 image on a CPU), itself tied to the pinned oracle on CPU and on two benchmark images;
  * threshold -> erode (+ add_dropped_objects) -> label -> dilate and the watershed: bit-exact against post_oracle;
  * scores: math.fsum per instance, 1e-10 relative (fp64 atomics add at most 90 000 terms in any order).

Measured on an H100 80GB HBM3 at its 700 W power limit: the CRF of the 64 benchmark tiles deviates from the float64
reference by at most 7.1e-5 and on average by 1.5e-8, so the CRF bar stays at max-abs 1e-4.  The whole file takes
about 55 s there."""
import math

import numpy as np
import pytest
import torch
from scipy import ndimage as ndi

import bench_data
from oracle import post_oracle as P

CRF_BAR = 1e-4
# crf.cu refuses kernel widths whose heaviest dropped tap, exp(-7^2 / (2 sxy^2)), exceeds 1e-7
SXY_MAX = 7.0 / math.sqrt(2.0 * math.log(1e7))


# ---------------------------------------------------------------------------------------------------------------------
# plain references
# ---------------------------------------------------------------------------------------------------------------------
def crf_rgb_ref(imgs):
    """post_oracle.crf_rgb_image for a batch: (N,3,H,W) float -> (N,H,W,3) uint8 (float64, truncate, wrap modulo 256)"""
    x = imgs.to(torch.float64)
    mean = torch.tensor(P.MEAN, dtype=torch.float64, device=x.device).view(1, 3, 1, 1)
    std = torch.tensor(P.STD, dtype=torch.float64, device=x.device).view(1, 3, 1, 1)
    v = ((x * std + mean) * 255.0).to(torch.int64) & 255
    return v.to(torch.uint8).permute(0, 2, 3, 1).contiguous()


def dense_crf_ref(imgs, probs, compat_gaussian=3.0, sxy_gaussian=1.0, compat_bilateral=10.0, sxy_bilateral=1.0,
                  srgb=50.0, iterations=5, radius=6):
    """post_oracle.dense_crf in float64 for a batch (N,3,H,W) / (N,2,H,W) on any device: exact Gaussian taps inside a
    (2 radius + 1)^2 window, symmetric normalisation, `iterations` mean-field updates -> (N,2,H,W) float64"""
    f = torch.float64
    n, _, h, w = probs.shape
    r = radius
    rgb = crf_rgb_ref(imgs).permute(0, 3, 1, 2).to(f)
    logp = torch.log(torch.clamp(probs.to(f), min=1e-5))

    def pad(a):
        return torch.nn.functional.pad(a, (r, r, r, r))

    def sh(a, dy, dx):   # a[y + dy, x + dx] of the padded array
        return a[:, :, r + dy:r + dy + h, r + dx:r + dx + w]

    inside = pad(torch.ones((n, 1, h, w), dtype=f, device=probs.device))
    rgb_p = pad(rgb)
    offs = [(dy, dx) for dy in range(-r, r + 1) for dx in range(-r, r + 1)]

    def kernels(dy, dx):
        d2 = float(dy * dy + dx * dx)
        m = sh(inside, dy, dx)
        col = torch.exp(-0.5 * ((rgb - sh(rgb_p, dy, dx)) ** 2).sum(1, keepdim=True) / (srgb * srgb))
        return math.exp(-0.5 * d2 / sxy_gaussian ** 2) * m, math.exp(-0.5 * d2 / sxy_bilateral ** 2) * col * m

    sg = torch.zeros((n, 1, h, w), dtype=f, device=probs.device)
    sb = torch.zeros_like(sg)
    for dy, dx in offs:
        kg, kb = kernels(dy, dx)
        sg += kg
        sb += kb
    ng, nb = 1.0 / torch.sqrt(sg + 1e-20), 1.0 / torch.sqrt(sb + 1e-20)
    q = torch.softmax(logp, dim=1)
    for _ in range(iterations):
        qg, qb = pad(q * ng), pad(q * nb)
        mg, mb = torch.zeros_like(q), torch.zeros_like(q)
        for dy, dx in offs:
            kg, kb = kernels(dy, dx)
            mg += kg * sh(qg, dy, dx)
            mb += kb * sh(qb, dy, dx)
        q = torch.softmax(logp + compat_gaussian * mg * ng + compat_bilateral * mb * nb, dim=1)
    return q


def fsum_scores(labels, prob, k):
    """build_score of one plane with exactly rounded sums: [(mean * sqrt(area)) or nan for labels 1..k]"""
    flat, pf = labels.ravel(), prob.ravel().astype(np.float64)
    order = np.argsort(flat, kind="stable")
    bounds = np.searchsorted(flat[order], np.arange(1, k + 2))
    out = []
    for i in range(k):
        vals = pf[order[bounds[i]:bounds[i + 1]]].tolist()
        c = len(vals)
        out.append(math.fsum(vals) / c * math.sqrt(c) if c else math.nan)
    return np.array(out)


def assert_scores(got, labels, prob, k):
    ref = fsum_scores(labels, prob, k)
    assert got.shape == ref.shape
    assert np.array_equal(np.isnan(got), np.isnan(ref))
    ok = ~np.isnan(ref)
    rel = np.abs(got[ok] - ref[ok]) / np.abs(ref[ok])
    assert rel.size == 0 or rel.max() <= 1e-10, rel.max()


def blob_map(rs, h, w, sigma):
    z = ndi.gaussian_filter(rs.randn(h, w), sigma)
    return ((z - z.min()) / (z.max() - z.min())).astype(np.float32)


def crf_inputs(n, h, w, seed):
    """n different images (N(0,1) noise plus a step where the building probability is high) and building-like soft
    maps, made like bench_data.probability_maps but for any (h, w)"""
    rs = np.random.RandomState(seed)
    p1 = []
    for _ in range(n):
        m, _ = bench_data.rectangles_mask(rs, h, w, 8)
        z = ndi.gaussian_filter(rs.randn(h, w) * 0.5 - 2.0 + 5.0 * m, 1.0)
        p1.append(1.0 / (1.0 + np.exp(-z)))
    p1 = np.stack(p1).astype(np.float32)
    probs = np.stack([1 - p1, p1], axis=1)
    imgs = (rs.randn(n, 3, h, w) + 1.5 * (p1[:, None] > 0.5)).astype(np.float32)
    return imgs, probs


def serpentine(h, w):
    """a 1-pixel corridor snaking row by row (every other row, joined alternately at the right and left ends)"""
    m = np.zeros((h, w), bool)
    rows = list(range(1, h - 1, 2))
    for j, y in enumerate(rows):
        m[y, 1:w - 1] = True
        if j + 1 < len(rows):
            m[y + 1, w - 2 if j % 2 == 0 else 1] = True
    return m, rows


# ---------------------------------------------------------------------------------------------------------------------
# CPU self-check of the float64 CRF reference against the pinned numpy oracle
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("h,w", [(40, 40), (23, 41)])
def test_dense_crf_reference_matches_oracle(h, w):
    imgs, probs = crf_inputs(2, h, w, seed=h + w)
    probs[0, 1, 3:7, 4:12], probs[0, 0, 3:7, 4:12] = 0.0, 1.0
    got = dense_crf_ref(torch.from_numpy(imgs), torch.from_numpy(probs)).numpy()
    for i in range(2):
        assert np.array_equal(crf_rgb_ref(torch.from_numpy(imgs[i:i + 1]))[0].numpy(), P.crf_rgb_image(imgs[i]))
        assert np.abs(got[i] - P.dense_crf(imgs[i], probs[i])).max() < CRF_BAR
    assert np.abs(dense_crf_ref(torch.from_numpy(imgs), torch.from_numpy(probs), iterations=2, sxy_bilateral=0.8)[1]
                  .numpy() - P.dense_crf(imgs[1], probs[1], iterations=2, sxy_bilateral=0.8)).max() < CRF_BAR


def test_fsum_scores_matches_oracle():
    rs = np.random.RandomState(3)
    lab = P.label(rs.rand(40, 50) < 0.4)
    prob = rs.rand(40, 50)
    k = int(lab.max())
    _, ref = P.build_score(lab[None], prob[None])
    assert np.allclose(fsum_scores(lab, prob, k), np.array(ref[0], dtype=np.float64), rtol=1e-12, atol=0)


# ---------------------------------------------------------------------------------------------------------------------
# A. the benchmark's chain on its own inputs
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def G(mcb, cuda):
    from mcb200 import postprocessing
    return postprocessing


@pytest.fixture(scope="module")
def chain(G, cuda):
    """bench.py infer_line's post-processing at --size 320 --batch 64: centre crop (m0 = 10), dense CRF, the graphed
    MaskPostprocessor((300, 300), 'resize', erode 2, dilate 2) and watershed_split(hi=0.8, lo=0.5)"""
    x, _ = bench_data.train_batch(64, 320, seed=1234)
    syn = bench_data.probability_maps(64, 320, seed=7)
    m0 = 10
    img = torch.from_numpy(x).to(cuda)[:, :, m0:320 - m0, m0:320 - m0].contiguous()
    pc = torch.from_numpy(syn).to(cuda)[:, :, m0:320 - m0, m0:320 - m0].contiguous()
    refined = G.dense_crf_batch(img, pc)
    pp = G.MaskPostprocessor((300, 300), "resize", erode_selem_size=2, dilate_selem_size=2)
    labels, scores, counts, pr = [t.clone() for t in pp.run_device_graphed(refined)]
    ws = G.watershed_split(refined[:, 1].contiguous(), hi=0.8, lo=0.5)
    torch.cuda.synchronize()
    return dict(img=img, pc=pc, refined=refined, pp=pp, labels=labels, scores=scores, counts=counts, pr=pr, ws=ws)


@pytest.mark.gpu
def test_bench_crf_against_float64_reference(chain):
    ref = torch.cat([dense_crf_ref(chain["img"][i:i + 16], chain["pc"][i:i + 16]) for i in range(0, 64, 16)])
    dev = (chain["refined"].double() - ref).abs()
    print("CRF 64x300x300 vs float64: max %.3e mean %.3e" % (float(dev.max()), float(dev.mean())))
    assert float(dev.max()) <= CRF_BAR
    assert float((chain["refined"].double().sum(1) - 1).abs().max()) < 1e-6


@pytest.mark.gpu
def test_bench_crf_against_numpy_oracle(chain):
    """ties the float64 reference to the pinned (float32, windowed) oracle at the benchmark size"""
    for i in (0, 63):
        img, pc = chain["img"][i].cpu().numpy(), chain["pc"][i].cpu().numpy()
        ref = P.dense_crf(img, pc)
        assert np.abs(chain["refined"][i].cpu().numpy() - ref).max() <= CRF_BAR
        assert np.abs(dense_crf_ref(chain["img"][i:i + 1], chain["pc"][i:i + 1])[0].cpu().numpy() - ref).max() <= CRF_BAR


@pytest.mark.gpu
def test_bench_crf_rgb_bit_exact(G, chain, cuda):
    from mcb200 import _lib as L
    img = chain["img"]
    rgb = torch.empty((64, 300, 300, 3), dtype=torch.uint8, device=cuda)
    L.fcall("mcb_crf_rgb_from_normalized", img.data_ptr(), rgb.data_ptr(), 64, 300, 300)
    got = rgb.cpu().numpy()
    imgs = img.cpu().numpy()
    for i in range(64):
        assert np.array_equal(got[i], P.crf_rgb_image(imgs[i])), i


@pytest.mark.gpu
def test_bench_mask_chain_bit_exact(chain):
    refined = chain["refined"].cpu().numpy()
    pr, labels = chain["pr"].cpu().numpy(), chain["labels"].cpu().numpy()
    counts = chain["counts"].cpu().numpy()
    for i in range(64):
        assert np.array_equal(pr[i], P.resize_image(refined[i], (300, 300))), i
        lab = P.label_multilayer_image(P.erode_image(P.categorize_multilayer_image(pr[i]), 2))
        assert np.array_equal(labels[i], P.dilate_image(lab, 2)), i
        assert np.array_equal(counts[2 * i:2 * i + 2], lab.reshape(2, -1).max(1)), i


@pytest.mark.gpu
def test_bench_scores_against_fsum(chain):
    labels = chain["labels"].view(128, 300, 300).cpu().numpy()
    pr = chain["pr"].view(128, 300, 300).cpu().numpy()
    counts, scores = chain["counts"].cpu().numpy(), chain["scores"].cpu().numpy()
    assert counts.max() <= scores.shape[1]
    for p in range(128):
        assert_scores(scores[p, :counts[p]], labels[p], pr[p], int(counts[p]))


@pytest.mark.gpu
def test_bench_watershed_split_bit_exact(chain):
    prob = chain["refined"][:, 1].cpu().numpy()
    ws = chain["ws"].cpu().numpy()
    for i in range(64):
        ref = P.minimax_watershed(prob[i], P.label(prob[i] > 0.8), prob[i] > 0.5)
        assert np.array_equal(ws[i], ref), (i, int((ws[i] != ref).sum()))


@pytest.mark.gpu
def test_bench_graph_replays_identical(chain):
    a = [t.clone() for t in chain["pp"].run_device_graphed(chain["refined"])]
    b = chain["pp"].run_device_graphed(chain["refined"])
    for x, y in ((a, b), (a, [chain["labels"], None, chain["counts"]])):
        assert torch.equal(x[0], y[0]) and torch.equal(x[2], y[2])


# ---------------------------------------------------------------------------------------------------------------------
# B. CRF edges
# ---------------------------------------------------------------------------------------------------------------------
def _crf_check(G, cuda, imgs, probs, radius=6, **kw):
    i, p = torch.from_numpy(imgs).to(cuda), torch.from_numpy(probs).to(cuda)
    got = G.dense_crf_batch(i, p, **kw)
    ref = dense_crf_ref(i, p, radius=radius, **kw)
    dev = (got.double() - ref).abs().amax(dim=(1, 2, 3)).cpu().numpy()
    assert dev.max() <= CRF_BAR, dev
    return got


@pytest.mark.gpu
@pytest.mark.parametrize("h,w", [(300, 200), (200, 300), (45, 301), (1, 40), (40, 1), (1, 1), (5, 77), (77, 5),
                                 (12, 12), (12, 45), (33, 65)])
def test_crf_shapes(G, cuda, h, w):
    """non-square images, images smaller than the 6-pixel halo, widths off the 32 grid; three different images per
    batch so that a wrong per-image offset shows"""
    imgs, probs = crf_inputs(3, h, w, seed=h * 1000 + w)
    _crf_check(G, cuda, imgs, probs)


@pytest.mark.gpu
@pytest.mark.parametrize("iterations", [1, 10])
def test_crf_iterations(G, cuda, iterations):
    imgs, probs = crf_inputs(2, 70, 90, seed=iterations)
    _crf_check(G, cuda, imgs, probs, iterations=iterations)


@pytest.mark.gpu
def test_crf_exact_zero_and_one_probabilities(G, cuda):
    imgs, probs = crf_inputs(2, 64, 64, seed=5)
    probs[:, 1, 10:30, 5:40], probs[:, 1, 40:60, 20:64] = 1.0, 0.0
    probs[:, 0] = 1.0 - probs[:, 1]
    _crf_check(G, cuda, imgs, probs)


@pytest.mark.gpu
def test_crf_without_pairwise_terms_is_the_clipped_input(G, cuda):
    imgs, probs = crf_inputs(2, 50, 70, seed=6)
    probs[:, 1, :10], probs[:, 1, 10:20] = 1.0, 0.0
    probs[:, 0] = 1.0 - probs[:, 1]
    got = G.dense_crf_batch(torch.from_numpy(imgs).to(cuda), torch.from_numpy(probs).to(cuda), compat_gaussian=0,
                            compat_bilateral=0, iterations=3).cpu().numpy().astype(np.float64)
    c = np.maximum(probs.astype(np.float64), np.float64(np.float32(1e-5)))
    ref = c / c.sum(1, keepdims=True)
    # logf / expf of exponents down to ln(1e-5) = -11.5: measured at most 8 float32 ulps
    ulp = np.spacing(ref.astype(np.float32)).astype(np.float64)
    assert (np.abs(got - ref) <= 8 * ulp).all(), (np.abs(got - ref) / ulp).max()


@pytest.mark.gpu
def test_crf_refuses_kernel_wider_than_its_window(G, cuda):
    """below the bound the windowed kernel matches a full-window filter; above it the call is refused -- at sxy = 1.3
    the 13x13 window would already move these outputs by more than the CRF bar"""
    x, _ = bench_data.train_batch(2, 64, seed=1)
    probs = bench_data.probability_maps(2, 64, seed=11, n_rect=8)
    i, p = torch.from_numpy(x).to(cuda), torch.from_numpy(probs).to(cuda)
    sxy_ok = math.floor(SXY_MAX * 100) / 100   # 1.23
    for kw in (dict(sxy_gaussian=sxy_ok), dict(sxy_bilateral=sxy_ok), dict(sxy_gaussian=sxy_ok, sxy_bilateral=sxy_ok)):
        got = G.dense_crf_batch(i, p, **kw)
        assert float((got.double() - dense_crf_ref(i, p, radius=8, **kw)).abs().max()) <= CRF_BAR, kw
    window = dense_crf_ref(i, p, sxy_gaussian=1.3, sxy_bilateral=1.3)
    assert float((window - dense_crf_ref(i, p, sxy_gaussian=1.3, sxy_bilateral=1.3, radius=8)).abs().max()) > CRF_BAR
    for kw in (dict(sxy_gaussian=sxy_ok + 0.01), dict(sxy_bilateral=sxy_ok + 0.01), dict(sxy_bilateral=3.0)):
        with pytest.raises(RuntimeError, match="too wide"):
            G.dense_crf_batch(i, p, **kw)
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------------------------------
# C. watershed edges
# ---------------------------------------------------------------------------------------------------------------------
def _ws_check(G, cuda, prob, markers, mask, levels=256):
    got = G.watershed_batch(torch.from_numpy(prob).to(cuda), torch.from_numpy(markers).to(cuda),
                            torch.from_numpy(mask).to(cuda), levels).cpu().numpy()
    for i in range(prob.shape[0]):
        ref = P.minimax_watershed(prob[i], markers[i], mask[i], levels)
        assert np.array_equal(got[i], ref), (i, int((got[i] != ref).sum()))
    return got


@pytest.mark.gpu
def test_watershed_more_than_1024_tiles(G, cuda):
    """33 x 32 tiles: the tile-activity table is off and every sweep visits every tile"""
    rs = np.random.RandomState(0)
    prob = blob_map(rs, 1056, 1000, 1.5)[None]
    got = _ws_check(G, cuda, prob, P.label(prob[0] > 0.65)[None].astype(np.int32), prob > 0.5)
    assert got.max() > 100


@pytest.mark.gpu
def test_watershed_serpentine_corridor(G, cuda):
    """a 1-pixel corridor ~4 400 steps long: far beyond the 128 relaxation steps of one tile visit, and it crosses the
    3 x 3 tiles both along and against each sweep direction, so tiles must be revisited across sweeps"""
    h = w = 96
    corridor, rows = serpentine(h, w)
    rs = np.random.RandomState(1)
    prob = np.where(corridor, 0.3 + 0.7 * rs.rand(h, w), 0.0).astype(np.float32)
    markers = np.zeros((3, h, w), np.int32)
    markers[0, rows[0], 1] = 5                       # one marker at the corridor's start ...
    markers[1, rows[-1], 1 if len(rows) % 2 == 0 else w - 2] = 5   # ... or at its end
    markers[2, rows[0], 1], markers[2, rows[-1], w // 2], markers[2, rows[20], 40] = 3, 9, 2
    got = _ws_check(G, cuda, np.stack([prob] * 3), markers, np.stack([corridor] * 3))
    assert (got[0][corridor] == 5).all() and (got[1][corridor] == 5).all()
    assert set(np.unique(got[2][corridor])) == {2, 3, 9}


@pytest.mark.gpu
@pytest.mark.parametrize("levels", [2, 65536])
def test_watershed_levels(G, cuda, levels):
    rs = np.random.RandomState(levels % 97)
    prob = np.stack([blob_map(rs, 70, 90, 3.0) for _ in range(3)])
    markers = np.stack([P.label(p > 0.75) for p in prob]).astype(np.int32)
    _ws_check(G, cuda, prob, markers, prob > 0.35, levels)


@pytest.mark.gpu
def test_watershed_float64_probabilities(G, cuda):
    rs = np.random.RandomState(2)
    prob = np.stack([blob_map(rs, 80, 75, 3.0) for _ in range(3)]).astype(np.float64)
    prob += rs.rand(*prob.shape) * 1e-9      # values a float32 copy would not keep
    markers = np.stack([P.label(p > 0.7) for p in prob]).astype(np.int32)
    _ws_check(G, cuda, prob, markers, prob > 0.4)


@pytest.mark.gpu
def test_watershed_64_planes_stray_markers_and_empty_masks(G, cuda):
    rs = np.random.RandomState(3)
    prob = np.stack([blob_map(rs, 48, 40, 2.5) for _ in range(64)])
    markers = np.stack([P.label(p > 0.75) for p in prob]).astype(np.int32)
    mask = prob > 0.4
    for i in range(0, 64, 4):                  # markers outside the mask
        ys, xs = rs.randint(0, 48, 6), rs.randint(0, 40, 6)
        markers[i, ys, xs] = rs.randint(1, 50, 6)
    mask[5] = False                           # markers, but an empty mask
    markers[6] = 0                            # a mask, but no markers
    got = _ws_check(G, cuda, prob, markers, mask)
    assert np.array_equal(got[5][markers[5] > 0], markers[5][markers[5] > 0]) and (got[6] == 0).all()


@pytest.mark.gpu
def test_watershed_large_marker_labels(G, cuda):
    """any positive int32 marker label survives, including those at and above the internal cost sentinel 2^30 - 1"""
    rs = np.random.RandomState(4)
    prob = np.stack([blob_map(rs, 64, 64, 3.0) for _ in range(2)])
    base = np.stack([P.label(p > 0.7) for p in prob])
    big = np.array([0, 2 ** 31 - 1, 0x3fffffff, 0x40000000, 7, 2 ** 31 - 2, 123456789, 0x3ffffffe, 2 ** 30 + 12345],
                   np.int64)
    lut = np.concatenate([big, rs.randint(1, 2 ** 31 - 1, max(0, int(base.max()) + 1 - big.size))])
    markers = lut[base].astype(np.int32)
    got = _ws_check(G, cuda, prob, markers, prob > 0.35)
    present = set(np.unique(markers)) - {0}
    assert {2 ** 31 - 1, 0x3fffffff, 0x40000000} <= present and set(np.unique(got)) - {0} == present


# ---------------------------------------------------------------------------------------------------------------------
# D. labelling, scores and morphology edges
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("dtype", ["uint8", "int32"])
@pytest.mark.parametrize("h,w", [(40, 308), (33, 512), (37, 1280), (1, 1280), (1, 308), (33, 300)])
def test_ccl_wide_planes_and_strip_borders(G, cuda, h, w, dtype):
    """widths above 307 need more than 48 KB of shared memory per strip; height 1 is a one-row strip, height 33 puts
    one row behind a strip border; the int32 path labels every nonzero value"""
    rs = np.random.RandomState(h + w)
    m = (rs.rand(3, h, w) < 0.55)
    if dtype == "int32":
        m = np.where(m, rs.randint(-5, 6, m.shape) | 1, 0).astype(np.int32)
    else:
        m = m.astype(np.uint8)
    lab, cnt = G.label_batch(torch.from_numpy(m).to(cuda), return_counts=True)
    ref = np.stack([P.label(x != 0) for x in m])
    assert np.array_equal(lab.cpu().numpy(), ref)
    assert np.array_equal(cnt.cpu().numpy(), ref.reshape(3, -1).max(1))


@pytest.mark.gpu
def test_ccl_refuses_width_beyond_strip(G, cuda):
    m = torch.zeros((1, 4, 1281), dtype=torch.uint8, device=cuda)
    with pytest.raises(RuntimeError, match="too large"):
        G.label_batch(m)


@pytest.mark.gpu
def test_transform_reruns_scores_beyond_kcap(G, cuda):
    """salt noise at 30 % gives ~4 900 / ~11 700 components per layer after erode 2: the scores are re-run with a
    larger kcap, and every instance, including the one at label == kcap, gets its exact score"""
    rs = np.random.RandomState(5)
    salt = rs.rand(2, 300, 300) < 0.3
    p1 = np.where(salt, 0.55 + 0.45 * rs.rand(2, 300, 300), 0.45 * rs.rand(2, 300, 300)).astype(np.float32)
    probs = np.stack([1 - p1, p1], axis=1)
    out = G.MaskPostprocessor((300, 300), "resize", erode_selem_size=2, dilate_selem_size=2).transform(probs)["y_pred"]
    for p, (labels, scores) in zip(probs, out):
        r = P.resize_image(p, (300, 300))
        lab = P.label_multilayer_image(P.erode_image(P.categorize_multilayer_image(r), 2))
        ref = P.dilate_image(lab, 2)
        assert np.array_equal(labels, ref)
        assert lab.max() > 1024
        for layer in range(2):
            k = int(lab[layer].max())
            got = np.array([math.nan if v is np.ma.masked else float(v) for v in scores[layer]])
            assert_scores(got, ref[layer], r[layer], k)


@pytest.mark.gpu
@pytest.mark.parametrize("size", [8, 16, 31])
def test_morphology_large_windows(G, cuda, size):
    probs = bench_data.probability_maps(2, 300, seed=size, n_rect=30)
    m = (probs > 0.5).astype(np.uint8).reshape(4, 300, 300)
    lab = np.stack([P.label(x) for x in m])
    d = G.morph_batch(torch.from_numpy(lab).to(cuda), size, True).cpu().numpy()
    assert np.array_equal(d, np.stack([P.dilate_image(x, size) for x in lab]))
    d8 = G.morph_batch(torch.from_numpy(m).to(cuda), size, True).cpu().numpy()
    assert np.array_equal(d8, np.stack([P.dilate_image(x, size) for x in m]))
    e = G.morph_batch(torch.from_numpy(m).to(cuda), size, False).cpu().numpy()
    assert np.array_equal(e, np.stack([P.skimage_erosion(x, P.skimage_rectangle(size, size)) for x in m]))
    ed = G.erode_batch(torch.from_numpy(m).to(cuda), size).cpu().numpy()
    assert np.array_equal(ed, np.stack([P.erode_image(x != 0, size) for x in m]))


@pytest.mark.gpu
@pytest.mark.parametrize("size", [0, 32])
def test_morph_rect_refuses_sizes(G, cuda, size):
    from mcb200 import _lib as L
    x = torch.zeros((1, 8, 8), dtype=torch.uint8, device=cuda)
    y = torch.empty_like(x)
    with pytest.raises(RuntimeError, match="size"):
        L.fcall("mcb_morph_rect", x.data_ptr(), y.data_ptr(), 0, 1, size, 1, 8, 8)
    torch.cuda.synchronize()
