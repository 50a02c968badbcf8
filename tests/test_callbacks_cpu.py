"""Drop-in boundary of mcb200.callbacks without a GPU: callbacks_unet builds from the reference's callbacks_config
keys (src/pipeline_config.py:93-118), and the monitor's validation_loss entry is what the reference's ModelCheckpoint /
EarlyStopping read (`val_loss['sum'].data.cpu().numpy()[0]`, src/steps/pytorch/callbacks.py:183,238)."""
import sys
import types

import numpy as np
import pytest
import torch

CALLBACKS_CONFIG = {     # src/pipeline_config.py:93-118 with neptune.yaml's values
    'model_checkpoint': {'filepath': '/tmp/checkpoints/unet/best.torch', 'epoch_every': 1, 'minimize': False},
    'exp_lr_scheduler': {'gamma': 0.9, 'epoch_every': 1},
    'plateau_lr_scheduler': {'lr_factor': 0.3, 'lr_patience': 30, 'epoch_every': 1},
    'training_monitor': {'batch_every': 1, 'epoch_every': 1},
    'experiment_timing': {'batch_every': 10, 'epoch_every': 1},
    'validation_monitor': {'epoch_every': 1, 'data_dir': '/data', 'validate_with_map': 1,
                           'small_annotations_size': 14},
    'neptune_monitor': {'model_name': 'unet', 'image_nr': 16, 'image_resize': 0.2,
                        'outputs_to_plot': ['multichannel_map']},
    'early_stopping': {'patience': 30, 'minimize': False},
}


class _Recorder:
    def __init__(self, **kwargs):
        self.kwargs = kwargs


def _reference_stand_in(monkeypatch):
    """`src.steps.pytorch.callbacks` / `src.callbacks` with the reference's constructor signatures"""
    def cls(name, params):
        def __init__(self, **kwargs):
            extra = [k for k in kwargs if k not in params]
            missing = [p for p in REQUIRED.get(name, ()) if p not in kwargs]
            assert not extra and not missing, (name, extra, missing)
            self.kwargs = kwargs
        return type(name, (), {"__init__": __init__})

    REQUIRED = {"ModelCheckpoint": ("filepath",), "ExponentialLRScheduler": ("gamma",), "EarlyStopping": ("patience",),
                "NeptuneMonitorSegmentation": ("image_nr", "image_resize", "model_name", "outputs_to_plot")}
    cb = types.ModuleType("src.steps.pytorch.callbacks")
    cb.ExperimentTiming = cls("ExperimentTiming", ("epoch_every", "batch_every"))
    cb.ModelCheckpoint = cls("ModelCheckpoint", ("filepath", "epoch_every", "minimize"))
    cb.ExponentialLRScheduler = cls("ExponentialLRScheduler", ("gamma", "epoch_every", "batch_every"))
    cb.TrainingMonitor = cls("TrainingMonitor", ("epoch_every", "batch_every"))
    cb.EarlyStopping = cls("EarlyStopping", ("patience", "minimize"))

    class CallbackList:
        def __init__(self, callbacks=None):
            self.callbacks = callbacks
    cb.CallbackList = CallbackList
    top = types.ModuleType("src.callbacks")
    top.NeptuneMonitorSegmentation = cls("NeptuneMonitorSegmentation",
                                         ("image_nr", "image_resize", "model_name", "outputs_to_plot"))
    for name, mod in (("src", types.ModuleType("src")), ("src.steps", types.ModuleType("src.steps")),
                      ("src.steps.pytorch", types.ModuleType("src.steps.pytorch")), ("src.steps.pytorch.callbacks", cb),
                      ("src.callbacks", top)):
        monkeypatch.setitem(sys.modules, name, mod)


def test_callbacks_unet_builds_from_the_reference_config(mcb, monkeypatch):
    from mcb200 import callbacks as C
    _reference_stand_in(monkeypatch)
    cl = C.callbacks_unet(CALLBACKS_CONFIG)
    names = [type(c).__name__ for c in cl.callbacks]
    assert names == ["ExperimentTiming", "TrainingMonitor", "ValidationMonitorSegmentation", "ModelCheckpoint",
                     "ExponentialLRScheduler", "EarlyStopping", "NeptuneMonitorSegmentation"]
    mon = cl.callbacks[2]
    assert isinstance(mon, C.ValidationMonitorSegmentation)
    assert mon.data_dir == '/data' and mon.small_annotations_size == 14 and mon.validate_with_map == 1
    assert mon.epoch_every == 1 and mon.target_size == (300, 300)


def test_monitor_validation_loss_is_what_checkpoint_and_early_stopping_read(mcb):
    from mcb200 import callbacks as C
    mon = C.ValidationMonitorSegmentation(data_dir='/data', small_annotations_size=14, validate_with_map=True,
                                          epoch_every=1)
    net = torch.nn.Identity()
    transformer = types.SimpleNamespace(model=net, optimizer=None, loss_function=None, output_names=['m'],
                                        validation_loss={})
    mon.set_params(transformer, validation_datagen=([], None), meta_valid=[1, 2])
    assert mon.validation_loss is transformer.validation_loss
    mon.on_train_begin()
    # an AP already stored for the epoch is returned as is (setdefault), without evaluating again
    transformer.validation_loss[0] = {'sum': torch.tensor([0.25])}
    mon.on_epoch_end()
    val = transformer.validation_loss[0]
    assert set(val) == {'sum'} and val['sum'].data.cpu().numpy()[0] == np.float32(0.25)
    assert mon.epoch_id == 1
    # epoch_every = 0 disables the validation, like the reference
    off = C.ValidationMonitorSegmentation('/data', 14, True, epoch_every=0)
    assert off.epoch_every is False


def test_monitor_falls_back_to_the_loss_without_map(mcb, monkeypatch):
    from mcb200 import callbacks as C
    calls = []
    val = types.ModuleType("src.steps.pytorch.validation")
    val.score_model = lambda model, loss_function, datagen: calls.append(1) or {'sum': torch.tensor([1.5])}
    for name in ("src", "src.steps", "src.steps.pytorch"):
        monkeypatch.setitem(sys.modules, name, types.ModuleType(name))
    monkeypatch.setitem(sys.modules, "src.steps.pytorch.validation", val)
    mon = C.ValidationMonitorSegmentation('/data', 14, validate_with_map=False, epoch_every=1)
    transformer = types.SimpleNamespace(model=torch.nn.Identity(), optimizer=None, loss_function=[], output_names=[],
                                        validation_loss={})
    mon.set_params(transformer, validation_datagen=([], None))
    mon.on_train_begin()
    mon.on_epoch_end()
    assert calls == [1] and transformer.validation_loss[0]['sum'].item() == 1.5
