"""TEST INFRASTRUCTURE — not part of the product path.

Imports the UNMODIFIED reference package (the `src` package of a checkout named by MCB_REFERENCE_ROOT, read-only) under Python 3.12 / torch 2.11 by
installing stub modules for its absent third-party dependencies (SURVEY.md Appendix B).  Used ONLY in the build
container, by oracle/make_golden.py (to generate tests/golden/*) and by the CPU tests that pin the oracle
restatements to the real reference.  Only the fixture generator (oracle/make_golden.py) imports this; no test does.

Stubs that carry behaviour (the skimage calls of src/postprocessing.py:4-5) delegate to oracle/post_oracle.py's
scipy restatements of skimage's documented implementation; everything else is inert.
"""
import collections
import collections.abc
import os
import sys
import tempfile
import types

REFERENCE_ROOT = os.environ.get("MCB_REFERENCE_ROOT", "")


def available():
    return bool(REFERENCE_ROOT) and os.path.isdir(os.path.join(REFERENCE_ROOT, "src"))


class _AttrDict(dict):
    """attrdict.AttrDict stand-in: recursive attribute access"""

    def __getattr__(self, k):
        try:
            v = self[k]
        except KeyError:
            raise AttributeError(k)
        return _AttrDict(v) if isinstance(v, dict) and not isinstance(v, _AttrDict) else v

    def __setattr__(self, k, v):
        self[k] = v

    def __getitem__(self, k):
        v = dict.__getitem__(self, k)
        return _AttrDict(v) if isinstance(v, dict) and not isinstance(v, _AttrDict) else v

    def get(self, k, d=None):
        return self[k] if k in self else d


class _Inert:
    """any attribute / call returns another inert object"""

    def __init__(self, *a, **k):
        pass

    def __getattr__(self, k):
        return _Inert()

    def __call__(self, *a, **k):
        return _Inert()


def _module(name, **attrs):
    m = types.ModuleType(name)
    m.__dict__.update(attrs)
    m.__getattr__ = lambda k: _Inert  # any other name resolves to the inert class
    sys.modules[name] = m
    return m


_installed = False


def install():
    """make `import src...` (the reference package) work; idempotent"""
    global _installed
    if _installed:
        return
    if not available():
        raise RuntimeError("reference tree not found at %s" % REFERENCE_ROOT)
    import torch  # noqa: F401  (before any stub)
    import torchvision  # noqa: F401
    import scipy.ndimage  # noqa: F401
    import scipy.stats  # noqa: F401
    import pandas  # noqa: F401
    import sklearn.ensemble  # noqa: F401
    import sklearn.model_selection  # noqa: F401
    import sklearn.metrics  # noqa: F401
    import joblib
    import yaml

    sys.dont_write_bytecode = True
    collections.Iterable = collections.abc.Iterable
    _orig_load = yaml.load
    if not getattr(yaml.load, "_mcb_patched", False):
        def _load(stream, Loader=None, **kw):
            return _orig_load(stream, Loader=Loader or yaml.FullLoader, **kw)
        _load._mcb_patched = True
        yaml.load = _load

    from . import post_oracle as P
    from . import instances_oracle as I

    _module("attrdict", AttrDict=_AttrDict)
    ext = _module("sklearn.externals", joblib=joblib)
    sys.modules["sklearn.externals.joblib"] = joblib
    import sklearn
    sklearn.externals = ext
    _module("neptune")
    _module("pydot_ng")
    _module("IPython")
    _module("IPython.display")
    _module("lightgbm")
    _module("xgboost")
    ia = _module("imgaug")
    iaa = _module("imgaug.augmenters")
    ia.augmenters = iaa
    sk = _module("skimage")
    sk.transform = _module("skimage.transform", resize=P.skimage_resize, rotate=I.skimage_rotate)
    sk.morphology = _module("skimage.morphology", erosion=P.skimage_erosion, dilation=P.skimage_dilation,
                            rectangle=P.skimage_rectangle)
    pd = _module("pydensecrf")
    pd.densecrf = _module("pydensecrf.densecrf")
    pd.utils = _module("pydensecrf.utils")
    pc = _module("pycocotools")
    pc.mask = _module("pycocotools.mask")
    pc.coco = _module("pycocotools.coco")
    _module("imageio")
    try:
        import cv2  # noqa: F401
    except Exception:
        _module("cv2")

    os.environ.setdefault("CONFIG_PATH", os.path.join(REFERENCE_ROOT, "neptune.yaml"))
    os.environ.setdefault("NEPTUNE_API_TOKEN", "x")
    if REFERENCE_ROOT not in sys.path:
        sys.path.insert(0, REFERENCE_ROOT)
    _installed = True


def reference_modules():
    """-> (src.unet_models, src.models, src.postprocessing, src.utils) of the real reference"""
    install()
    import src.unet_models as um
    import src.models as mo
    import src.postprocessing as pp
    import src.utils as ut
    for cfg in mo.PRETRAINED_NETWORKS.values():
        if "pretrained" in cfg["model_config"]:
            cfg["model_config"]["pretrained"] = False  # no network for ImageNet weights
    return um, mo, pp, ut


def reference_unet_config(encoder="ResNet34", image_hw=(256, 256)):
    """the `config.unet` dict of src/pipeline_config.py:61-120 with experiment dirs pointed at a temp dir"""
    install()
    import src.pipeline_config as pc
    cfg = pc.SOLUTION_CONFIG["unet"]

    def plain(d):
        return {k: plain(v) if isinstance(v, dict) else v for k, v in d.items()}

    cfg = plain(cfg)
    cfg["architecture_config"]["model_params"]["encoder"] = encoder
    cfg["architecture_config"]["weighted_cross_entropy"]["imsize"] = tuple(image_hw)
    tmp = tempfile.mkdtemp(prefix="mcb_ref_")
    cb = cfg["callbacks_config"]
    cb["model_checkpoint"]["filepath"] = os.path.join(tmp, "checkpoints", "unet", "best.torch")
    return cfg
