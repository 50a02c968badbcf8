"""Drop-in boundary (SURVEY.md 8b): the surface the reference's callbacks and checkpoint round trips touch.  No GPU:
nothing is computed."""
import pytest
import torch


def test_fit_loop_metrics_shape_suits_the_reference_callbacks():
    """TrainingMonitor.on_batch_end does loss.data.cpu().numpy()[0] (src/steps/pytorch/callbacks.py:134): the step's
    metric must be a 1-element 1-D tensor (a 0-d tensor raises IndexError there)"""
    import inspect
    import mcb200  # noqa: F401
    from mcb200 import models as mm
    src = inspect.getsource(mm.FusedTrainStep.step)
    assert "reshape(1)" in src
    assert torch.zeros(()).reshape(1).clone().data.cpu().numpy()[0] == 0.0


def test_arena_survives_device_noops_and_rebuilds_on_moves():
    """ADVICE r1: `.cuda()` on a model that is already there (save_model's round trip ends with it, _to_device runs every
    batch) must keep arenas / plans; a real move re-packs them and bumps the generation the fused step checks"""
    import mcb200  # noqa: F401
    from mcb200.unet_models import UNetResNet
    net = UNetResNet(34, 2, 32, 0.0, False, True)
    gen, p32 = net._generation, net._p32
    net.float()                        # nothing moves
    net.to(torch.device("cpu"))
    assert net._generation == gen and net._p32 is p32 and net._params_alias_arena()
    w = net.final.weight
    assert w.data_ptr() == p32.data_ptr() + 4 * net._slots[id(w)].off
    with pytest.raises(AssertionError):    # a dtype move tears the views off; fp32 masters are required, said loudly
        net.double()
