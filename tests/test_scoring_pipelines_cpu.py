"""The reference's second-level scoring pipelines (src/pipelines.py:307-411) with mcb200.postprocessing as their `post`
module, and the pins of the scoring oracle (oracle/scoring_oracle.py).  No GPU: nothing is computed on a device.

* The four scoring pipelines (`scoring_model` train, `unet_scoring_model`, `unet_padded_scoring_model`,
  `unet_tta_scoring_model` inference) build from the unchanged src/pipelines.py with `post` bound to
  mcb200.postprocessing and a RandomForest scoring model (lightgbm is not installed).
* CATEGORY_LAYERS / CATEGORY_IDS come from the reference's src/pipeline_config.py when it is importable ([1, 19] once
  the scoring workflow sets it) and stay [1, 1] / [None, 100] without it.
* The oracle equals tests/golden/scoring_features.npz (the unmodified reference's output) bit for bit, and equals the
  reference live when the reference tree is present.

The reference is imported through oracle/ref_shim.py, which installs stub modules; each such check runs in a child
process so that the stubs never reach the other tests.
"""
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest

from oracle import ref_shim
from oracle import scoring_oracle as S

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "scoring_features.npz")
needs_reference = pytest.mark.skipif(not ref_shim.available(), reason="reference tree (MCB_REFERENCE_ROOT) absent")


def run_child(code, tmp_path):
    env = dict(os.environ, PYTHONPATH=ROOT, MCB_TMP=str(tmp_path))
    r = subprocess.run([sys.executable, "-c", textwrap.dedent(code)], cwd=ROOT, env=env, capture_output=True, text=True,
                       timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    return r.stdout


@needs_reference
def test_scoring_pipelines_build_with_the_dropin(tmp_path):
    out = run_child("""
        import os
        from oracle import ref_shim
        ref_shim.reference_modules()
        import mcb200
        from mcb200 import postprocessing as post
        import src.pipeline_config as cfg
        import src.pipelines as pl
        pl.post = post                                   # INTEGRATION.md 2b: `from mcb200 import postprocessing as post`
        cfg.CATEGORY_LAYERS = [1, 19]
        config = cfg.SOLUTION_CONFIG
        dict.__getitem__(config, 'env')['cache_dirpath'] = os.environ['MCB_TMP']
        dict.__getitem__(config, 'postprocessor')['scoring_model'] = 'rf'
        for name in ('scoring_model', 'unet_scoring_model', 'unet_padded_scoring_model', 'unet_tta_scoring_model'):
            mode = 'train' if name == 'scoring_model' else 'inference'
            pipe = pl.PIPELINES[name][mode](config)
            fe = pipe.get_step('feature_extractor').transformer
            assert isinstance(fe, post.FeatureExtractor), name
            sm = pipe.get_step('scoring_model').transformer
            assert type(sm).__name__ == 'ScoringRandomForest', name
            if mode == 'inference':
                assert isinstance(pipe.get_step('score_builder').transformer, post.ScoreImageJoiner)
                assert isinstance(pipe.get_step('nms').transformer, post.NonMaximumSupression)
            print(name, 'built')
        assert post.get_thresholds() == post.layer_thresholds([1, 19])[0] and len(post.get_thresholds()) == 20
    """, tmp_path)
    assert out.count("built") == 4


@needs_reference
def test_category_layers_follow_the_reference_config(tmp_path):
    run_child("""
        from oracle import ref_shim
        ref_shim.install()
        import mcb200
        from mcb200 import postprocessing as post
        import src.pipeline_config as cfg
        assert post.category_config() == ([1, 1], [None, 100])
        cfg.CATEGORY_LAYERS = [1, 19]
        layers, ids = post.category_config()
        assert layers == [1, 19] and ids == [None, 100]
        thr, chan = post.layer_thresholds()
        assert len(thr) == 20 and chan == [0] + [1] * 19
        assert [round(t, 2) for t in post.get_thresholds()] == [0.5] + [round(0.05 * k, 2) for k in range(1, 20)]
        assert post.MaskPostprocessor().category_layers == [1, 1]      # its explicit argument, as before
    """, tmp_path)


def test_category_layers_default_without_the_reference(tmp_path):
    run_child("""
        import sys
        import mcb200
        from mcb200 import postprocessing as post
        assert 'src' not in sys.modules
        assert post.category_config() == ([1, 1], [None, 100])
        assert post.get_thresholds() == [0.5, 0.5] and post.layer_thresholds()[1] == [0, 1]
    """, tmp_path)


def test_category_layers_warn_when_the_reference_config_fails(tmp_path):
    """a `src` package whose pipeline_config does not import: the defaults, said loudly"""
    (tmp_path / "src").mkdir()
    (tmp_path / "src" / "__init__.py").write_text("")
    (tmp_path / "src" / "pipeline_config.py").write_text("raise KeyError('CONFIG_PATH')\n")
    run_child("""
        import os, sys, warnings
        sys.path.insert(0, os.environ['MCB_TMP'])
        import mcb200
        from mcb200 import postprocessing as post
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter('always')
            assert post.category_config() == ([1, 1], [None, 100])
        assert any(issubclass(x.category, RuntimeWarning) and 'pipeline_config' in str(x.message) for x in w)
    """, tmp_path)


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLD)


def assert_flat_equal(got, golden, prefix):
    for k, v in got.items():
        want = golden["%s_%s" % (prefix, k)]
        if v.dtype.kind == "f":
            assert np.array_equal(v, want, equal_nan=True), k
        else:
            assert np.array_equal(v, want), k


def test_oracle_matches_golden(golden):
    """the restatement on the golden's inputs (20 images, [1, 19]) is the reference's output bit for bit, dtypes
    included"""
    probs, labels, annotations = S.scoring_case()
    got = S.flatten(S.feature_extractor(list(labels), list(probs), annotations)['features'])
    assert_flat_equal(got, golden, "ann")
    assert golden["ann_counts"].size == 20 * 20 and golden["ann_counts"].sum() > 1000
    # the case's corners: no annotations on image 0, none above 0.5 on image 2, iou None on every background layer
    none = golden["ann_iou_none"].reshape(20, 20)
    counts = golden["ann_counts"].reshape(20, 20)
    assert none[0][counts[0] > 0].all() and none[:, 0][counts[:, 0] > 0].all()
    assert (counts[2, 10:] == 0).all() and not none[1:, 1:][counts[1:, 1:] > 0].any()
    iou = golden["ann_iou"]
    assert np.nanmax(iou) > 0.9 and (iou == 0).any()


def test_oracle_without_annotations_matches_golden(golden):
    probs, labels, _ = S.scoring_case()
    idx = [0, 2, 7]
    got = S.flatten(S.feature_extractor(list(labels[idx]), list(probs[idx]))['features'])
    rows = golden["none_counts"].reshape(20, 20)
    starts = np.concatenate([[0], np.cumsum(golden["none_counts"])])
    sel = np.concatenate([np.arange(starts[i * 20], starts[(i + 1) * 20]) for i in idx])
    for k, v in got.items():
        if k in ("counts", "iou_none", "dtypes"):
            assert np.array_equal(v, golden["none_" + k].reshape(20, 20)[idx].reshape(-1)), k
        else:
            assert np.array_equal(v, golden["none_" + k][sel], equal_nan=True), k
    assert rows.sum() == golden["ann_counts"].sum()


@needs_reference
def test_oracle_matches_the_reference_live(tmp_path):
    """a small fresh case (4 images of 64 x 64) through the unmodified reference and through the restatement"""
    run_child("""
        import copy
        from oracle import make_golden_scoring as M
        from oracle import scoring_oracle as S
        pp = M.reference_postprocessing()
        probs, labels, annotations = S.scoring_case(n=4, size=64, seed=5)
        want = pp.FeatureExtractor().transform(list(labels), list(probs), copy.deepcopy(annotations))['features']
        got = S.feature_extractor(list(labels), list(probs), annotations)['features']
        M.frames_equal(got, want)
        assert sum(len(df) for im in got for df in im) > 20
    """, tmp_path)


def test_golden_tells_the_first_polygon_from_all_polygons(golden, monkeypatch):
    """merging every polygon of a segmentation (instead of frPyObjects(...)[0]) changes `iou` on the golden's inputs:
    the instance-aligned annotations carry the instance's box as a second polygon after a decoy"""
    from oracle import overlay_oracle as OV
    probs, labels, annotations = S.scoring_case()
    idx = [3, 4, 5]

    def merged(segm, h, w):
        return {"size": [h, w], "counts": OV.ann_to_rle(segm, h, w)}

    monkeypatch.setattr(S, "first_segmentation_rle", merged)
    got = S.flatten(S.feature_extractor(list(labels[idx]), list(probs[idx]), [annotations[i] for i in idx])['features'])
    starts = np.concatenate([[0], np.cumsum(golden["ann_counts"])])
    sel = np.concatenate([np.arange(starts[i * 20], starts[(i + 1) * 20]) for i in idx])
    want = golden["ann_iou"][sel]
    assert np.array_equal(np.isnan(got["iou"]), np.isnan(want))
    assert (got["iou"][~np.isnan(want)] != want[~np.isnan(want)]).sum() >= 5
    assert (golden["ann_iou"] > 0.5).sum() > 100
