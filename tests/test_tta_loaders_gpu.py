"""GPU parity of the TTA inference loaders (src/loaders.py:74-111,307-398,477-487; csrc/instances.cu
tta_variants_u8_kernel through mcb200.loaders): the colour kernel bit-identical to cv2 on every colour, every geometry
code against oracle/tta_oracle.py, the loaders end to end from PNG files against the oracle rows built with the flow's
own draws, and the unet_tta chain (loader -> network -> aggregator) against the oracle batches."""
import numpy as np
import pytest
import torch

from oracle import instances_oracle as I
from oracle import tta_oracle as T

pytestmark = pytest.mark.gpu


def _variants(tiles, src, codes, cuda):
    """the kernel alone: uint8 variant rows (NV, H, W, 3) on the device"""
    from mcb200 import _lib as L
    x = torch.from_numpy(np.ascontiguousarray(tiles)).to(cuda)
    n, h, w, _ = x.shape
    out = torch.empty((len(codes), h, w, 3), dtype=torch.uint8, device=cuda)
    src_d = torch.from_numpy(np.asarray(src, np.int32)).to(cuda)
    codes_d = torch.from_numpy(np.asarray(codes, np.int32)).to(cuda)
    L.fcall("mcb_tta_variants_u8", x.data_ptr(), out.data_ptr(), src_d.data_ptr(), codes_d.data_ptr(), len(codes), h, w)
    return out


def test_colour_kernel_equals_cv2_on_every_colour(mcb, cuda):
    """all 2^24 colours as one 4096 x 4096 image (a multiple of every cv2 vector width: every pixel takes cv2's vector
    body), each of the six branches at every value 0..100, compared on the device"""
    import cv2
    from mcb200 import _lib as L
    idx = np.arange(1 << 24, dtype=np.uint32)
    rgb = np.stack([idx >> 16, (idx >> 8) & 255, idx & 255], -1).astype(np.uint8).reshape(4096, 4096, 3)
    hsv = cv2.cvtColor(rgb, cv2.COLOR_RGB2HSV)
    x = torch.from_numpy(rgb).to(cuda)[None]
    src = torch.zeros(1, dtype=torch.int32, device=cuda)
    out = torch.empty_like(x)
    for branch in range(1, 7):
        c = (branch - 1) % 3
        base = hsv if branch <= 3 else rgb
        chan = np.ascontiguousarray(base[..., c])
        for value in range(101):
            shifted = base.copy()
            shifted[..., c] = cv2.add(chan, value)                    # saturating: Add + clip at 255
            want = cv2.cvtColor(shifted, cv2.COLOR_HSV2RGB) if branch <= 3 else shifted
            code = torch.tensor([branch << 4 | value << 8], dtype=torch.int32, device=cuda)
            L.fcall("mcb_tta_variants_u8", x.data_ptr(), out.data_ptr(), src.data_ptr(), code.data_ptr(), 1, 4096, 4096)
            bad = (out[0] != torch.from_numpy(want).to(cuda)).any(-1)
            assert not bool(bad.any()), (branch, value, int(bad.sum()))


def test_every_geometry_code_with_colour(mcb, cuda):
    rs = np.random.RandomState(8)
    tiles = rs.randint(0, 256, (2, 300, 300, 3)).astype(np.uint8)
    codes, src, want = [], [], []
    for k in range(4):
        for flip in range(3):
            for branch in range(7):
                value = int(rs.randint(0, 101))
                t = int(rs.randint(0, 2))
                img = tiles[t] if branch == 0 else T.color_shift(tiles[t], branch, value, tail=False)
                img = np.flipud(img) if flip == 1 else (np.fliplr(img) if flip == 2 else img)
                want.append(np.rot90(img, k))
                codes.append(k | flip << 2 | branch << 4 | value << 8)
                src.append(t)
    got = _variants(tiles, src, codes, cuda).cpu().numpy()
    for g, w, c in zip(got, want, codes):
        assert np.array_equal(g, w), c


def _png_tiles(tmp_path, n=6, size=300, seed=12):
    from PIL import Image
    rs = np.random.RandomState(seed)
    paths, tiles = [], []
    for i in range(n):
        # smooth colour fields plus noise: every HSV sector and saturation range occurs
        yy, xx = np.mgrid[0:size, 0:size] / size
        base = np.stack([np.sin(6 * xx + i), np.cos(5 * yy - i), np.sin(4 * (xx + yy))], -1) * 100 + 128
        img = np.clip(base + rs.randint(-30, 31, base.shape), 0, 255).astype(np.uint8)
        p = str(tmp_path / ("tile%d.png" % i))
        Image.fromarray(img).save(p)
        paths.append(p)
        tiles.append(np.array(Image.open(p).convert('RGB')))
    return paths, tiles


PARAMS = {'inference': {'batch_size': 20, 'shuffle': False, 'num_workers': 0, 'pin_memory': False}}
DATASET = {'h': 256, 'w': 256, 'h_pad': 10, 'w_pad': 10}


def _oracle_row(tile, spec, draw, mode, tail):
    return T.tta_loader_row(tile, spec, draw, mode, pad=(10, 10), size=(256, 256), tail=tail)


def _run_flow(flow):
    """iterate a flow, keeping every batch and its draws"""
    batches, draws = [], []
    for X in flow:
        batches.append(X)
        draws.append(flow.last_draws)
    return batches, draws


@pytest.mark.parametrize("runs", [False, 2])
@pytest.mark.parametrize("mode", ["resize", "crop_and_pad"])
def test_tta_loaders_end_to_end(mcb, cuda, tmp_path, monkeypatch, runs, mode):
    from mcb200 import loaders as lo
    paths, tiles = _png_tiles(tmp_path)
    decodes = []
    orig = lo.SegmentationFiles.__getitem__
    monkeypatch.setattr(lo.SegmentationFiles, "__getitem__", lambda self, i: (decodes.append(i), orig(self, i))[1])
    gen = lo.TestTimeAugmentationGenerator(flip_ud=True, flip_lr=True, rotation=True, color_shift_runs=runs)
    meta = gen.transform(np.array(paths)[:, None])
    params, ids = meta['tta_params'], meta['img_ids']
    X = np.asarray(meta['X_tta'].values)[:, 0]                        # squeeze_inputs, src/utils.py:227-228
    Loader = lo.ImageSegmentationLoaderResizeTTA if mode == "resize" else lo.ImageSegmentationLoaderInferencePaddingTTA
    flow, steps = Loader(PARAMS, DATASET, seed=3).transform(X, params)['datagen']
    batches, draws = _run_flow(flow)
    nrows = 6 * (33 if runs else 16)
    assert len(decodes) == 6 and steps == len(batches) == -(-nrows // 20)
    assert [len(b) for b in batches[:-1]] == [20] * (steps - 1) and len(batches[-1]) == nrows - 20 * (steps - 1)
    hw = 256 if mode == "resize" else 320
    excepted, colour_rows, row = 0, 0, 0
    for b, d in zip(batches, draws):
        assert b.shape[1:] == (3, hw, hw) and b.dtype == torch.float32 and b.is_cuda
        got = b.cpu().numpy()
        for i in range(len(b)):
            spec, tile = params[row], tiles[ids[row]]
            colour = T.applies_colour(spec)
            assert (d['branch'][i] != 0) == colour and (1 <= d['branch'][i] <= 6 or not colour)
            draw = (int(d['branch'][i]), int(d['value'][i])) if colour else None
            want = _oracle_row(tile, spec, draw, mode, tail=False)
            assert np.array_equal(got[i], want), (row, spec, draw)
            if colour:
                colour_rows += 1
                ref = _oracle_row(tile, spec, draw, mode, tail=True)     # cv2's scalar tail columns as the reference
                excepted += int((got[i] != ref).any(0).sum())
            row += 1
    assert row == nrows and colour_rows == (6 * 8 if runs else 0)
    print("%s runs=%s: %d colour rows, %d pixels excepted for cv2's scalar-tail columns" % (mode, runs, colour_rows,
                                                                                          excepted))
    # a second pass decodes every file once more and draws afresh
    _run_flow(flow)
    assert len(decodes) == 12


def test_inference_padding_matches_the_pad_chain(mcb, cuda, tmp_path):
    from mcb200 import loaders as lo
    paths, tiles = _png_tiles(tmp_path, seed=13)
    flow, steps = lo.ImageSegmentationLoaderInferencePadding(PARAMS, DATASET).transform(np.array(paths))['datagen']
    batches, _ = _run_flow(flow)
    assert steps == 1 and batches[0].shape == (6, 3, 320, 320)
    got = batches[0].cpu().numpy()
    for g, t in zip(got, tiles):
        assert np.array_equal(g, _oracle_row(t, None, None, "crop_and_pad", tail=False))


def test_unet_tta_pipeline_with_colour(mcb, cuda, tmp_path):
    """loader -> PyTorchUNet.transform -> TestTimeAugmentationAggregator: the probabilities equal the same net's on the
    oracle-built batches, the aggregate is within 2e-6 of the reference's inverse transforms + scipy gmean"""
    import bench
    from mcb200 import loaders as lo
    from mcb200.models import PyTorchUNet
    from oracle import unet_oracle as O
    paths, tiles = _png_tiles(tmp_path, seed=14)
    model = PyTorchUNet(**bench.unet_config("ResNet34"))
    model.model.load_state_dict(O.make_reference_like_state_dict(34, seed=11))
    model._to_device()
    meta = lo.TestTimeAugmentationGenerator(flip_ud=True, flip_lr=True, rotation=True,
                                            color_shift_runs=2).transform(np.array(paths)[:, None])
    params, ids = meta['tta_params'], meta['img_ids']
    flow, steps = lo.ImageSegmentationLoaderResizeTTA(PARAMS, DATASET, seed=5).transform(
        np.asarray(meta['X_tta'].values)[:, 0], params)['datagen']
    draws = []

    def recorded():
        for X in flow:
            draws.append(flow.last_draws)
            yield X

    (probs,) = model.transform((recorded(), steps)).values()
    assert probs.shape == (6 * 33, 2, 256, 256) and len(draws) == steps
    oracle_batches, row = [], 0
    for d in draws:
        rows = []
        for i in range(len(d['branch'])):
            draw = (int(d['branch'][i]), int(d['value'][i])) if d['branch'][i] else None
            rows.append(_oracle_row(tiles[ids[row]], params[row], draw, "resize", tail=False))
            row += 1
        oracle_batches.append(torch.from_numpy(np.stack(rows)).to(cuda))
    (want_probs,) = model.transform((oracle_batches, steps)).values()
    assert np.array_equal(probs, want_probs)
    agg = lo.TestTimeAugmentationAggregator('gmean', 1).transform(probs, params, ids)['aggregated_prediction']
    want = I.tta_aggregate(list(probs), params, ids, 'gmean')
    assert len(agg) == 6
    for a, b in zip(agg, want):
        assert a.shape == b.shape == (2, 256, 256) and np.abs(a - b).max() < 2e-6
