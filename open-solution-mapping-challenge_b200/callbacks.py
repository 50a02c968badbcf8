"""The validation callback of the reference (src/callbacks.py:108-200) with its mAP computed on the device.

Per validation batch everything stays on the H100: eval forward -> softmax -> resize to the 300 x 300 target size ->
argmax -> label every class -> build_score -> `DeviceCOCOEvaluator.add_batch`; after the last batch one `result()`.
The reference instead stacks every logit on the host, post-processes image by image, writes a result JSON and runs
the vendored COCOeval on it.

In `crop_and_pad` mode the reference's callback resizes the 320 x 320 prediction to 300 x 300 and does not crop it
(its target size is fixed, src/callbacks.py:187); so does this one.

Under torch.distributed every rank evaluates the whole validation set; replicas are identical, so is the AP.

Opt in with `callbacks=mcb200.callbacks.callbacks_unet(config.unet.callbacks_config)`.
"""
import logging
import os

import numpy as np
import torch

from . import ops
from .evaluation import CATEGORY_IDS, CATEGORY_LAYERS, DeviceCOCOEvaluator
from .postprocessing import categorize_batch, label_batch, resize_batch, scores_strided

logger = logging.getLogger(__name__)
Y_COLUMNS_SCORING = ['ImageId']   # src/pipeline_config.py:16


class ValidationMonitorSegmentation:
    """src/callbacks.py:108-125 (constructor, set_params) and src/steps/pytorch/callbacks.py:147-167 (epoch_every,
    on_epoch_end).  The epoch's AP is stored as transformer.validation_loss[epoch_id] = {'sum': tensor([AP])}, which
    is what the reference's ModelCheckpoint and EarlyStopping read."""

    def __init__(self, data_dir, small_annotations_size, validate_with_map=False, epoch_every=None, batch_every=None,
                 target_size=(300, 300)):
        self.epoch_id = None
        self.batch_id = None
        self.model = self.optimizer = self.loss_function = self.output_names = self.validation_datagen = None
        self.epoch_every = False if epoch_every == 0 else epoch_every
        self.batch_every = False if batch_every == 0 else batch_every
        self.data_dir = data_dir
        self.small_annotations_size = small_annotations_size
        self.validate_with_map = validate_with_map
        self.target_size = tuple(target_size)
        self.validation_loss = None
        self.meta_valid = None
        self._evaluator = None

    def set_params(self, transformer, validation_datagen, meta_valid=None, *args, **kwargs):
        self.model = transformer.model
        self.optimizer = transformer.optimizer
        self.loss_function = transformer.loss_function
        self.output_names = transformer.output_names
        self.validation_datagen = validation_datagen
        self.meta_valid = meta_valid
        self.validation_loss = transformer.validation_loss

    # ---- Callback surface (src/steps/pytorch/callbacks.py:13-60)
    def on_train_begin(self, *args, **kwargs):
        self.epoch_id = 0
        self.batch_id = 0

    def on_train_end(self, *args, **kwargs):
        pass

    def on_epoch_begin(self, *args, **kwargs):
        pass

    def on_batch_begin(self, *args, **kwargs):
        pass

    def on_batch_end(self, *args, **kwargs):
        self.batch_id += 1

    def training_break(self, *args, **kwargs):
        return False

    def on_epoch_end(self, *args, **kwargs):
        if self.epoch_every and ((self.epoch_id % self.epoch_every) == 0):
            self.model.eval()
            val_loss = self.get_validation_loss()
            self.model.train()
            for name, loss in val_loss.items():
                logger.info('epoch {0} validation {1}:     {2:.5f}'.format(self.epoch_id, name,
                                                                          loss.data.cpu().numpy()[0]))
        self.epoch_id += 1

    def get_validation_loss(self):
        if self.validate_with_map:
            return self._get_validation_loss()
        if self.epoch_id not in self.validation_loss.keys():   # the reference's loss-based validation
            from src.steps.pytorch.validation import score_model
            self.validation_loss[self.epoch_id] = score_model(self.model, self.loss_function, self.validation_datagen)
        return self.validation_loss[self.epoch_id]

    # ---- mAP on the device
    def evaluator(self):
        """the ground truth of the validation set as device tables, built on first use"""
        if self._evaluator is None:
            image_ids = np.asarray(self.meta_valid[Y_COLUMNS_SCORING[0]].values if hasattr(self.meta_valid, 'columns')
                                   else self.meta_valid)
            self._evaluator = DeviceCOCOEvaluator(os.path.join(self.data_dir, 'val', 'annotation.json'), image_ids,
                                                  list(CATEGORY_IDS[1:]), self.small_annotations_size,
                                                  CATEGORY_IDS, CATEGORY_LAYERS)
        return self._evaluator

    def _get_validation_loss(self):
        if self.epoch_id in self.validation_loss:      # setdefault: the first value of an epoch stays
            return self.validation_loss[self.epoch_id]
        ev = self.evaluator()
        ev.reset()
        ids = np.asarray(self.meta_valid[Y_COLUMNS_SCORING[0]].values if hasattr(self.meta_valid, 'columns')
                         else self.meta_valid)
        batch_gen, steps = self.validation_datagen
        net = self.model
        dev = ev.device
        seen = 0
        with torch.no_grad():
            for batch_id, data in enumerate(batch_gen):
                X = data[0] if isinstance(data, (list, tuple)) else data
                logits = net(X.to(dev).float())
                self.add_logits(logits, ids[seen:seen + logits.shape[0]])
                seen += logits.shape[0]
                if batch_id == steps:
                    break
        if ev._next_id == 1:                            # no detections: 0 without evaluating (src/callbacks.py:137-138)
            ap = 0.0
        else:
            ap = float(ev.result()["ap_ar"][0])
        return self.validation_loss.setdefault(self.epoch_id, {'sum': torch.tensor([ap], dtype=torch.float32)})

    def add_logits(self, logits, image_ids):
        """one validation batch of logits (N, 2, H, W) -> softmax, resize, argmax, label, build_score, add_batch"""
        probs = ops.softmax2(logits.contiguous())
        pr = resize_batch(probs, self.target_size)
        cat = categorize_batch(pr)
        n, c, h, w = pr.shape
        planes = torch.stack([(cat == k) for k in range(c)], dim=1).to(torch.uint8).contiguous()
        labels, counts = label_batch(planes, return_counts=True)
        kcap = 1024
        while True:
            scores = scores_strided(labels.view(n * c, h, w), pr.view(n * c, h, w), counts, kcap)
            top = int(counts.max())
            if top <= kcap:
                break
            kcap = top
        self.evaluator().add_batch(labels, scores, image_ids, counts)


def callbacks_unet(callbacks_config):
    """src/models.py:295-307 with this module's ValidationMonitorSegmentation in place of the reference's; the other
    callbacks are the reference's own (its `src` package must be importable)."""
    from src.steps.pytorch.callbacks import CallbackList, EarlyStopping, ExperimentTiming, \
        ExponentialLRScheduler, ModelCheckpoint, TrainingMonitor
    from src.callbacks import NeptuneMonitorSegmentation
    experiment_timing = ExperimentTiming(**callbacks_config['experiment_timing'])
    model_checkpoints = ModelCheckpoint(**callbacks_config['model_checkpoint'])
    lr_scheduler = ExponentialLRScheduler(**callbacks_config['exp_lr_scheduler'])
    training_monitor = TrainingMonitor(**callbacks_config['training_monitor'])
    validation_monitor = ValidationMonitorSegmentation(**callbacks_config['validation_monitor'])
    neptune_monitor = NeptuneMonitorSegmentation(**callbacks_config['neptune_monitor'])
    early_stopping = EarlyStopping(**callbacks_config['early_stopping'])
    return CallbackList(callbacks=[experiment_timing, training_monitor, validation_monitor, model_checkpoints,
                                   lr_scheduler, early_stopping, neptune_monitor])
