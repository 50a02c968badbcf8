"""The training augmentation on the H100 (csrc/augment.cu through mcb200.augmentation and mcb200.loaders) against the
CPU restatement of imgaug + skimage + Pillow + torchvision (oracle/augment_oracle.py): bit-exact."""
import os

import numpy as np
import pytest
import torch

from oracle import augment_oracle as AO
from oracle import synthetic

pytestmark = pytest.mark.gpu

H = W = 300
SEQUENCES = [(c,) for c in range(3)] + [(a, b) for a in range(3) for b in range(3) if a != b]   # the 9 child orders


def _batch(n, seed):
    """n 300x300 samples: images (some with a minimum above 0, so the warp's clip acts), 0/1 masks, distances and
    sizes above 255 (the uint16 -> uint8 wrap)"""
    rs = np.random.RandomState(seed)
    imgs = rs.randint(0, 256, (n, H, W, 3)).astype(np.uint8)
    imgs[::3] = np.maximum(imgs[::3], 37)
    masks = np.stack([synthetic.rectangles_mask(rs, H, W, n_rect=8, lo=6, hi=40)[0] for _ in range(n)]).astype(np.uint8)
    masks = (masks > 0).astype(np.uint8)
    dist = rs.randint(0, 1200, (n, H, W)).astype(np.uint16)
    dist[1::4] += 3                                              # minimum above 0 here too
    sizes = rs.randint(1, 700, (n, H, W)).astype(np.uint16)
    return imgs, masks, dist, sizes


def _params(n, crop, seed):
    from mcb200 import augmentation as A
    seq = A.crop_seq((256, 256)) if crop else A.fast_seq
    p = seq.draw(np.random.default_rng(seed), n, H, W)
    combos = [(children, coin) for children in SEQUENCES for coin in (True, False)][:n]
    for i, (children, coin) in enumerate(combos):
        p[i]['n_children'] = len(children)
        p[i]['children'] = list(children) + [-1] * (2 - len(children))
        p[i]['coin'] = coin
    return p


@pytest.mark.parametrize("crop", [False, True], ids=["resize", "crop"])
@pytest.mark.parametrize("with_distances", [True, False], ids=["distances", "mask"])
def test_batch32_bit_exact_against_oracle(mcb, cuda, crop, with_distances):
    from mcb200 import augmentation as A
    imgs, masks, dist, sizes = _batch(32, 11 + crop)
    p = _params(32, crop, 5 + crop)
    d, s = (dist, sizes) if with_distances else (None, None)
    crop_size = (256, 256) if crop else None
    img_u8, tgt_u8 = A.augment_batch(imgs, masks, d, s, p, crop_size)
    img_u8, tgt_u8 = img_u8.cpu().numpy(), tgt_u8.cpu().numpy()
    X, T = A.batch_chain(imgs, masks, d, s, p, crop_size=crop_size, resize=None if crop else (256, 256))
    X, T = X.cpu().numpy(), T.cpu().numpy()
    assert X.shape == (32, 3, 256, 256) and T.shape == (32, 3 if with_distances else 1, 256, 256)
    for i in range(32):
        mrgb = np.dstack([masks[i]] * 3)
        di, si = (dist[i], sizes[i]) if with_distances else (None, None)
        wi, wt = AO.augmented_planes(imgs[i], mrgb, di, si, p[i], crop_size)
        assert np.array_equal(img_u8[i], wi), (i, p[i])
        assert np.array_equal(tgt_u8[i], wt), (i, p[i])
        x, t = AO.loader_sample(imgs[i], mrgb, di, si, p[i], "crop" if crop else "resize", (256, 256))
        assert np.array_equal(X[i], x) and np.array_equal(T[i], t), (i, p[i])


def test_identity_parameters_reproduce_the_unaugmented_path(mcb, cuda):
    from mcb200 import augmentation as A
    from mcb200 import preparation as prep
    imgs, masks, _, _ = _batch(4, 3)
    rs = np.random.RandomState(4)
    dsum = (rs.rand(4, H, W) * 900).astype(np.float16)
    big = rs.randint(1, 90000, (4, H, W)).astype(np.int64)
    d16 = dsum.astype(np.uint16)
    s16 = np.sqrt(big.astype(np.uint16)).astype(np.uint16)
    ident = A.identity_params(4)
    X, T = A.batch_chain(imgs, masks, d16, s16, ident, resize=(256, 256))
    assert torch.equal(X, prep.image_transform_resize_batch(imgs, (256, 256)))
    X, T = A.batch_chain(imgs, masks, d16, s16, ident, pad=(10, 10))
    assert torch.equal(X, prep.image_transform_batch(imgs, (10, 10)))
    assert torch.equal(T, prep.target_batch(masks, dsum, big, (10, 10)))
    X, T = A.batch_chain(imgs, masks, None, None, ident)
    assert torch.equal(T[:, 0], torch.from_numpy(masks).to(cuda).float())


def test_bad_crops_and_parameter_rows_raise(mcb, cuda):
    from mcb200 import augmentation as A
    imgs, masks, dist, sizes = _batch(3, 6)
    p = _params(3, True, 1)
    with pytest.raises(ValueError):
        A.augment_batch(imgs, masks, dist, sizes, p[:2], (256, 256))          # one row per sample
    bad = p.copy()
    bad[1]['top'] = 300 - 256 + 1
    with pytest.raises(RuntimeError, match="crop"):
        A.augment_batch(imgs, masks, dist, sizes, bad, (256, 256))
    with pytest.raises(RuntimeError):
        A.augment_batch(imgs, masks, dist, sizes, A.identity_params(3), (320, 256))
    with pytest.raises(ValueError):
        A.augment_batch(imgs, masks, dist, None, p, (256, 256))
    with pytest.raises(ValueError):
        A.augment_batch(imgs, masks, dist.astype(np.int32), sizes, p, (256, 256))
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------ loaders from files
def _write_dataset(root, n, seed):
    """the reference's on-disk layout: images, masks/*.png, distances/* and sizes/* (joblib, no extension)"""
    import joblib
    from PIL import Image
    imgs, masks, _, _ = _batch(n, seed)
    rs = np.random.RandomState(seed)
    X, y = [], []
    for sub in ("images", "masks", "distances", "sizes"):
        os.makedirs(os.path.join(root, sub), exist_ok=True)
    for i in range(n):
        xp, mp = os.path.join(root, "images", "%d.png" % i), os.path.join(root, "masks", "%d.png" % i)
        Image.fromarray(imgs[i]).save(xp)
        Image.fromarray(masks[i]).save(mp)                                       # mode L, 0/1
        joblib.dump((rs.rand(H, W) * 1100).astype(np.float16), os.path.join(root, "distances", "%d" % i))
        sz = np.ones((H, W), np.int64)
        sz[masks[i] > 0] = rs.randint(1, 90000)
        joblib.dump(sz, os.path.join(root, "sizes", "%d" % i))
        X.append(xp)
        y.append(mp)
    return np.array(X), np.array(y)


def _reference_sample(X, y, i, distances):
    """what the reference's Dataset reads before its augmenter (src/loaders.py:141-154)"""
    import joblib
    from PIL import Image
    img = np.array(Image.open(X[i]).convert('RGB'))
    mrgb = np.array(Image.open(y[i]).convert('RGB'))
    if not distances:
        return img, mrgb, None, None
    dp = os.path.splitext(y[i].replace("/masks/", "/distances/"))[0]
    d = joblib.load(dp).astype(np.uint16)
    s = np.sqrt(joblib.load(dp.replace("/distances/", "/sizes/")).astype(np.uint16)).astype(np.uint16)
    return img, mrgb, d, s


LOADERS = ["MetadataImageSegmentationLoaderDistancesResize", "MetadataImageSegmentationLoaderDistancesCropPad",
           "MetadataImageSegmentationLoaderResize", "MetadataImageSegmentationLoaderCropPad"]


@pytest.mark.parametrize("name", LOADERS)
def test_loader_flows_bit_exact_with_partial_last_batch(mcb, cuda, tmp_path, name):
    from mcb200 import loaders
    X, y = _write_dataset(str(tmp_path), 5, 21)
    params = {'training': {'batch_size': 2, 'shuffle': False, 'num_workers': 2, 'pin_memory': True},
              'inference': {'batch_size': 2, 'shuffle': False, 'num_workers': 0, 'pin_memory': False}}
    dp = {'h': 256, 'w': 256, 'h_pad': 10, 'w_pad': 10}
    loader = getattr(loaders, name)(params, dp, seed=3)
    crop, distances = "CropPad" in name, "Distances" in name
    out = loader.transform(X, y, X, y)
    (flow, steps), (vflow, vsteps) = out['datagen'], out['validation_datagen']
    assert steps == 3 and vsteps == 3
    for flow_, train in ((flow, True), (vflow, False)):
        seen = 0
        for batch in flow_:
            assert isinstance(batch, list) and len(batch) == 2 and batch[0].is_cuda and batch[1].is_cuda
            n = batch[0].shape[0]
            assert n == (1 if seen == 4 else 2)                                   # the partial last batch
            side = 256 if (train or not crop) else 320
            assert batch[0].shape == (n, 3, side, side) and batch[1].shape == (n, 3 if distances else 1, side, side)
            for j in range(n):
                img, mrgb, d, s = _reference_sample(X, y, seen + j, distances)
                x, t = AO.loader_sample(img, mrgb, d, s, flow_.last_params[j] if train else None,
                                        "crop" if crop else "resize", (256, 256), train=train)
                assert np.array_equal(batch[0][j].cpu().numpy(), x), (name, train, seen + j)
                assert np.array_equal(batch[1][j].cpu().numpy(), t), (name, train, seen + j)
            seen += n
        assert seen == 5
    again = getattr(loaders, name)(params, dp, seed=3).transform(X, y)['datagen'][0]
    first = [b[0].clone() for b in again]
    assert all(torch.equal(a, b) for a, b in zip(first, [b[0] for b in loader.transform(X, y)['datagen'][0]]))


def test_fit_loop_on_loader_batches_matches_oracle_batches(mcb, cuda, tmp_path):
    """three PyTorchUNetWeighted._fit_loop steps (ResNet34, batch 2, 256x256) fed by the device loader give the losses
    and weights of the fused train step fed the oracle's host-built batches of the same draws (the step is bitwise
    deterministic)"""
    import bench
    from mcb200 import loaders
    from mcb200.models import PyTorchUNetWeighted
    X, y = _write_dataset(str(tmp_path), 6, 31)
    params = {'training': {'batch_size': 2, 'shuffle': False, 'num_workers': 0, 'pin_memory': True},
              'inference': {'batch_size': 2, 'shuffle': False, 'num_workers': 0}}
    loader = loaders.MetadataImageSegmentationLoaderDistancesResize(params, {'h': 256, 'w': 256}, seed=9)
    flow, _ = loader.transform(X, y)['datagen']
    with torch.random.fork_rng(devices=[cuda]):
        torch.manual_seed(0)
        a = PyTorchUNetWeighted(**bench.unet_config("ResNet34"))
        b = PyTorchUNetWeighted(**bench.unet_config("ResNet34"))
    b.model.load_state_dict(a.model.state_dict())
    losses_a, losses_b = [], []
    for k, batch in enumerate(flow):
        losses_a.append(a._fit_loop(batch)['sum'].detach().cpu().clone())
        xs, ts = [], []
        for j, idx in enumerate((2 * k, 2 * k + 1)):
            img, mrgb, d, s = _reference_sample(X, y, idx, True)
            x, t = AO.loader_sample(img, mrgb, d, s, flow.last_params[j], "resize", (256, 256))
            xs.append(x)
            ts.append(t)
        losses_b.append(b._fit_loop([torch.from_numpy(np.stack(xs)), torch.from_numpy(np.stack(ts))])['sum']
                        .detach().cpu().clone())
    assert len(losses_a) == 3
    assert all(torch.equal(p, q) for p, q in zip(losses_a, losses_b)), (losses_a, losses_b)
    sa, sb = a.model.state_dict(), b.model.state_dict()
    for k in sa:
        assert torch.equal(sa[k], sb[k]), k
