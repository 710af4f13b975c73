"""Train an LSTM model file to file on the device: the reference's trainer CLI (trajnetbaselines/lstm/trainer.py) over a
device-resident scene store.

    python -m trajnetplusplusbaselines_b200.lstm.trainer --path trajdata --type directional --augment --normalize_scene

The reference prepares every scene of every batch in Python (paths_to_xy, drop_distant, center_scene, random_rotation,
add_noise in NumPy, lstm/trainer.py:96-133) and syncs once per batch on `loss.item()`.  Here:

  * `prepare_data` reads every file through the native ndjson parser into one `SceneStore`: the float64 scenes
    [T, M_store, 2] on the device, drop_distant (r = 6) run once at load (it is deterministic per scene), so the host knows
    every batch's `batch_split` without a device sync;
  * `draw_epoch_plan` consumes Python's and NumPy's global generators exactly as `Trainer.train` does (one shuffle, one
    theta per scene, one start length per batch, one noise block per scene), up front;
  * one `tb2_scenes_gather_epoch` launch (csrc/scene_ops.cu) then builds every batch of the epoch, each a contiguous
    float32 [T, M_b, 2] block, bit-identical to `torch.Tensor(np.concatenate([...]))` of the reference's chain;
  * `train_batch` / `val_batch` keep the reference's computation; their losses stay on the device, and the host syncs only
    where the reference logs.

With the same seeds and the same scene list the batches, losses, parameters and optimizer state equal those of the
reference's `Trainer.loop` driving this package's model, bit for bit.  Only configurations the training backward supports
are accepted (`check_trainable`).
"""
import argparse
import json
import logging
import math
import os
import random
import socket
import sys
import time
from collections import OrderedDict

import numpy as np
import torch

from .. import _lib
from ..data import load_scenes_xy
from ..engine import _device_of, _ptr, _stream
from .gridbased_pooling import GridBasedPooling
from .loss import L2Loss, PredictionLoss
from .lstm import LSTM, LSTMPredictor
from .non_gridbased_pooling import (AttentionMLPPooling, HiddenStateMLPPooling, NearestNeighborLSTM, NearestNeighborMLP,
                                    TrajectronPooling)
from .scene_ops import _frame_table, scene_frames

DROP_DISTANT_R = 6.0          # drop_distant's default radius (lstm/lstm.py:16), the trainer's call (lstm/trainer.py:109)
NOISE_THRESH = 0.02           # add_noise(scene, thresh=0.02, ped='neigh') (lstm/trainer.py:118)
NOISE_FRAMES = 9              # add_noise's default obs_length: the trainer does not pass its own (augmentation.py:79)

GOALS_MESSAGE = "goal_flag=True is not built (off in every BASELINE config)"


class SceneStore(object):
    """The scenes of one set (train or val) on the device.

    entries: [(filename, scene_id, xy float64 [T, N_i, 2], primary first)], every scene with the same T.
    xy [T, M_store, 2] float64 and scene_off [n + 1] int32 live on `device`; drop_distant runs once here
    (`tb2_scenes_drop_distant`), leaving the keep mask and kept counts on the device and the kept counts on the host
    (`kept`).  The primaries' tracks stay on the host (`primary` [T, n, 2]) for center_scene's O(n) scalars."""

    def __init__(self, entries, device=None):
        self.T = int(entries[0][2].shape[0]) if entries else 0
        for f, sid, xy in entries:
            if xy.shape[0] != self.T:
                raise ValueError("%s: scene %s has %d frames, the scenes before it %d; every scene of a set must have the "
                                 "same frame count" % (f, sid, xy.shape[0], self.T))
        _lib.require_cuda()
        lib = _lib.load()
        self.device = _device_of(device)
        self.names = [(f, sid) for f, sid, _ in entries]
        self.n = len(entries)
        self.order = list(range(self.n))          # the scene list Trainer.train shuffles in place, epoch after epoch
        sizes = np.array([xy.shape[1] for _, _, xy in entries], dtype=np.int64)
        split = np.zeros(self.n + 1, dtype=np.int64)
        split[1:] = np.cumsum(sizes)
        self.split = split
        host = (np.ascontiguousarray(np.concatenate([xy for _, _, xy in entries], axis=1), dtype=np.float64)
                if entries else np.zeros((0, 0, 2)))
        self.primary = np.ascontiguousarray(host[:, split[:-1]])
        M = int(split[-1])
        self._frames = {}
        self._val = {}
        with torch.cuda.device(self.device):
            self.xy = torch.from_numpy(host).to(self.device)
            self.scene_off = torch.from_numpy(split.astype(np.int32)).to(self.device)
            self.keep = torch.empty(M, dtype=torch.uint8, device=self.device)
            self.kept_count = torch.zeros(self.n, dtype=torch.int32, device=self.device)
            if self.n:
                _lib.check(lib.tb2_scenes_drop_distant(_ptr(self.xy), _ptr(self.scene_off), self.T, M, self.n,
                                                       DROP_DISTANT_R ** 2, _ptr(self.keep), _ptr(self.kept_count),
                                                       _stream(self.device)))
            self.kept = self.kept_count.cpu().numpy().astype(np.int64)

    def __len__(self):
        return self.n

    @classmethod
    def from_files(cls, filenames, sample=1.0, device=None):
        """Every scene of every file, files in the given order, scenes in file order (data.load_scenes_xy).  sample < 1:
        `random.sample` of int(len * sample) scenes of each file, kept in file order."""
        entries = []
        for fn in filenames:
            name = os.path.basename(fn).split('.')[-2]
            scenes = load_scenes_xy(fn)
            T = entries[0][2].shape[0] if entries else (scenes[0][1].shape[0] if scenes else 0)
            for sid, xy in scenes:
                if xy.shape[0] != T:
                    raise ValueError("%s: scene %s has %d frames, the scenes before it %d; every scene of a set must "
                                     "have the same frame count" % (fn, sid, xy.shape[0], T))
            if sample != 1.0:
                picked = sorted(random.sample(range(len(scenes)), int(len(scenes) * sample)))
                scenes = [scenes[i] for i in picked]
            entries += [(name, sid, xy) for sid, xy in scenes]
        return cls(entries, device)

    def frames(self, obs_length):
        """[n, 4] float64 device table (centre x, centre y, cos, sin of the rotation) of center_scene per store scene."""
        table = self._frames.get(obs_length)
        if table is None:
            center, rotation = scene_frames(self.primary, np.arange(self.n + 1), obs_length)
            table = torch.from_numpy(_frame_table(center, rotation)).to(self.device)
            self._frames[obs_length] = table
        return table

    def gather(self, order, batch_size, frame=None, thetas=None, noise=None, noise_off=None):
        """The batches of `order` (store scene per position) in one tb2_scenes_gather_epoch launch.

        Returns [(batch_scene float32 [T, M_b, 2] view of one epoch buffer, batch_split int64 ndarray [B_b + 1])]."""
        lib = _lib.load()
        order = np.asarray(order, dtype=np.int64)
        n = len(order)
        counts = self.kept[order]
        bounds = list(range(0, n, batch_size)) + [n]
        tracks = np.array([int(counts[a:b].sum()) for a, b in zip(bounds[:-1], bounds[1:])], dtype=np.int64)
        base = np.zeros(len(tracks), dtype=np.int64)
        if len(tracks) > 1:
            base[1:] = np.cumsum(tracks[:-1]) * self.T
        total = int(tracks.sum()) * self.T
        d = self.device
        with torch.cuda.device(d):
            out = torch.empty(total * 2, dtype=torch.float32, device=d)
            if n:
                perm = torch.from_numpy(order.astype(np.int32)).to(d)
                base_d = torch.from_numpy(base).to(d)
                tracks_d = torch.from_numpy(tracks.astype(np.int32)).to(d)
                aug = None
                if thetas is not None:
                    aug = torch.from_numpy(np.ascontiguousarray(_frame_table(np.zeros((n, 2)), thetas)[:, 2:4])).to(d)
                noise_d = noise_off_d = None
                if noise is not None:
                    noise_d = torch.from_numpy(np.ascontiguousarray(noise, dtype=np.float64)).to(d)
                    noise_off_d = torch.from_numpy(np.asarray(noise_off, dtype=np.int64)).to(d)
                _lib.check(lib.tb2_scenes_gather_epoch(
                    _ptr(self.xy), _ptr(self.scene_off), _ptr(self.keep), _ptr(self.kept_count), self.T,
                    int(self.xy.shape[1]), _ptr(perm), n, int(batch_size), _ptr(base_d), _ptr(tracks_d), _ptr(frame),
                    _ptr(aug), _ptr(noise_d), _ptr(noise_off_d), min(NOISE_FRAMES, self.T), _ptr(out), _stream(d)))
        batches = []
        for k, (a, b) in enumerate(zip(bounds[:-1], bounds[1:])):
            lo = int(base[k]) * 2
            view = out[lo:lo + int(tracks[k]) * self.T * 2].view(self.T, int(tracks[k]), 2)
            split = np.zeros(b - a + 1, dtype=np.int64)
            split[1:] = np.cumsum(counts[a:b])
            batches.append((view, split))
        return batches

    def val_batches(self, batch_size, frame=None):
        """The validation batches (scenes in store order, no random draws): assembled once, reused every epoch."""
        key = (batch_size, None if frame is None else frame.data_ptr())
        if key not in self._val:
            self._val[key] = self.gather(np.arange(self.n), batch_size, frame=frame)
        return self._val[key]


class EpochPlan(object):
    """What one epoch of Trainer.train draws: order [n] (store scene per position), thetas [n] or None, start_lengths
    (one per batch) or None, noise (float64, one [9, kept - 1, 2] block per scene in position order) and noise_off [n]
    or None, and the batch splits."""

    def __init__(self, order, thetas, start_lengths, noise, noise_off, splits):
        self.order, self.thetas, self.start_lengths = order, thetas, start_lengths
        self.noise, self.noise_off, self.splits = noise, noise_off, splits


def draw_epoch_plan(order, kept, batch_size, n_frames, obs_length=9, augment=False, augment_noise=False,
                    obs_dropout=False):
    """Consume the global generators as Trainer.train does for one epoch (lstm/trainer.py:86-157, 248-250).

    `order` (a list, shuffled IN PLACE like the reference's scene list) -> EpochPlan.  Python's generator: one shuffle,
    then per scene in shuffled order one random.random() for theta (augment), and after the last scene of each batch one
    random.randint(0, obs_length - 2) (obs_dropout).  NumPy's global generator: add_noise's uniform(-0.02, 0.02) blocks of
    every scene in order, drawn as one array of the concatenated size (the same values)."""
    random.shuffle(order)
    n = len(order)
    thetas = [] if augment else None
    starts = [] if obs_dropout else None
    for i in range(n):
        if augment:
            thetas.append(random.random() * 2.0 * math.pi)
        if obs_dropout and ((i + 1) % batch_size == 0 or i + 1 == n):
            starts.append(random.randint(0, obs_length - 2))
    perm = np.asarray(order, dtype=np.int64)
    counts = np.asarray(kept, dtype=np.int64)[perm] if n else np.zeros(0, dtype=np.int64)
    noise = noise_off = None
    if augment_noise:
        sizes = min(NOISE_FRAMES, n_frames) * (counts - 1) * 2
        noise_off = np.zeros(n, dtype=np.int64)
        if n > 1:
            noise_off[1:] = np.cumsum(sizes)[:-1]
        noise = np.random.uniform(-NOISE_THRESH, NOISE_THRESH, int(sizes.sum()))
    splits = []
    for a in range(0, n, batch_size):
        split = np.zeros(len(counts[a:a + batch_size]) + 1, dtype=np.int64)
        split[1:] = np.cumsum(counts[a:a + batch_size])
        splits.append(split)
    return EpochPlan(perm, None if thetas is None else np.asarray(thetas, dtype=np.float64), starts, noise, noise_off,
                     splits)


def check_trainable(model):
    """Raise, with the message the training path itself would raise, for a model whose training backward is not built:
    goal_flag, the non-grid interaction modules, grid embeddings other than one_layer (two_layer too for social),
    constant != 0, pool widths above 1024, hidden_dim outside {32, 64, ..., 256}."""
    from .training import _grad_targets
    if model.goal_flag:
        raise NotImplementedError(GOALS_MESSAGE)
    _grad_targets(model)                          # NotImplementedError for the non-grid modules
    if model.hidden_dim not in _lib.HIDDEN_DIMS:
        raise RuntimeError(_lib.HIDDEN_DIM_MESSAGE)
    pool = model.pool
    if pool is None or not hasattr(pool, 'fill_config'):       # none, or an external module (trained through autograd)
        return
    layers = 0 if pool.embedding is None else sum(isinstance(m, torch.nn.Linear) for m in pool.embedding)
    width = pool.out_dim if layers else pool.n * pool.n * pool.pooling_dim
    if pool.type_ == 'social':
        if layers not in (1, 2) or not model.pool_to_input or pool.constant != 0:
            raise RuntimeError("social training backward supports one_layer / two_layer embeddings with constant = 0")
    elif layers != 1 or not model.pool_to_input or pool.constant != 0 or width > 1024:
        raise RuntimeError("training backward supports one_layer grid embeddings with constant = 0 and pool_to_input")


class Trainer(object):
    """The reference's Trainer (lstm/trainer.py:28-311) over SceneStore scene sets: same constructor arguments, same
    `loop / train / val / train_batch / val_batch`.  train_batch / val_batch take the reference's arguments and do its
    computation; they return the losses as device tensors (0-dim), which the loop reads back only where it logs.

    adv_eps > 0 adds adversarial training against the collision attack (attack.pgd_collision): every training batch
    first attacks its observation, each scene's primary moved inside a per-frame L2 ball of radius adv_eps (metres) by
    adv_steps PGD iterations, then trains on (1 - adv_wt) * clean loss + adv_wt * attacked loss.  The attack draws no
    random numbers, so the epoch plan is the one of a clean run.  adv_eps = 0 (the default) is the reference's
    computation.

    contrast_weight > 0 adds the Social-NCE term (lstm/contrast.py): every training batch trains on
    criterion * batch_size + contrast_weight * L_nce, the query being each primary's hidden state after the step that
    consumed the last observed frame.  `contrast` is the SocialNCE module (default: SocialNCE(model.hidden_dim), built
    after the model); its parameters join the optimizer.  The term draws its noise from torch's generator on the
    device, so the epoch plan is the one of a clean run; the epoch records gain `loss_nce`, the mean L_nce over the
    epoch's batches.  contrast_weight = 0 (the default) builds and draws nothing."""

    def __init__(self, model=None, criterion=None, optimizer=None, lr_scheduler=None,
                 device=None, batch_size=8, obs_length=9, pred_length=12, augment=True,
                 normalize_scene=False, save_every=1, start_length=0, obs_dropout=False,
                 augment_noise=False, val_flag=True, adv_eps=0.0, adv_steps=5, adv_wt=0.5,
                 contrast_weight=0.0, contrast=None):
        self.model = model if model is not None else LSTM()
        if not contrast_weight >= 0:
            raise ValueError("contrast_weight must be >= 0, got %r" % (contrast_weight,))
        self.contrast_weight = float(contrast_weight)
        self.contrast = None
        if self.contrast_weight > 0:
            if adv_eps > 0:
                raise ValueError("Social-NCE (contrast_weight > 0) together with adversarial training (adv_eps > 0) "
                                 "is not built")
            from .contrast import SocialNCE, check_contrast
            check_contrast(self.model)
            self.contrast = contrast if contrast is not None else SocialNCE(self.model.hidden_dim)
            if self.contrast.hidden_dim != self.model.hidden_dim:
                raise ValueError("the SocialNCE module is built for hidden_dim %d, the model has %d"
                                 % (self.contrast.hidden_dim, self.model.hidden_dim))
            if not 1 <= self.contrast.horizon <= pred_length:
                raise ValueError("the Social-NCE horizon must be in [1, pred_length = %d], got %d"
                                 % (pred_length, self.contrast.horizon))
        self.criterion = criterion if criterion is not None else PredictionLoss()
        self.optimizer = optimizer if optimizer is not None else \
            torch.optim.Adam(self.model.parameters(), lr=1e-3, weight_decay=1e-4)
        if self.contrast is not None:
            known = {id(p) for group in self.optimizer.param_groups for p in group['params']}
            heads = [p for p in self.contrast.parameters() if id(p) not in known]
            if heads:
                self.optimizer.add_param_group({'params': heads})
        self.lr_scheduler = lr_scheduler if lr_scheduler is not None else \
            torch.optim.lr_scheduler.StepLR(self.optimizer, 15)

        self.device = device if device is not None else torch.device('cuda')
        self.model = self.model.to(self.device)
        self.criterion = self.criterion.to(self.device)
        if self.contrast is not None:
            self.contrast = self.contrast.to(self.device)
        self.log = logging.getLogger(self.__class__.__name__)
        self.save_every = save_every

        self.batch_size = batch_size
        self.obs_length = obs_length
        self.pred_length = pred_length
        self.seq_length = self.obs_length + self.pred_length

        self.augment = augment
        self.augment_noise = augment_noise
        self.normalize_scene = normalize_scene

        self.start_length = start_length
        self.obs_dropout = obs_dropout

        self.val_flag = val_flag
        if not adv_eps >= 0:
            raise ValueError("adv_eps must be >= 0, got %r" % (adv_eps,))
        if adv_eps > 0:
            if int(adv_steps) != adv_steps or adv_steps < 1:
                raise ValueError("adv_steps must be an integer >= 1, got %r" % (adv_steps,))
            if not 0 < adv_wt <= 1:
                raise ValueError("adv_wt must be in (0, 1], got %r" % (adv_wt,))
            from .training import check_rollout
            check_rollout(self.model)         # NotImplementedError for the models the attack cannot differentiate
        self.adv_eps, self.adv_steps, self.adv_wt = float(adv_eps), int(adv_steps), float(adv_wt)
        self._col_counts = None           # [clean, attacked] scenes with D <= 0.2 m this epoch (adv_eps > 0), on the device
        self._start_lengths = None        # the epoch plan's obs_dropout draws, consumed by train_batch
        self._nce_losses = None           # this epoch's L_nce per batch (contrast_weight > 0), on the device
        self._zeros = torch.zeros((0, 2), device=self.device)

    def _goals(self, num_tracks):
        """The all-zero goals the reference builds per batch (lstm/trainer.py:106); the model does not read them."""
        if self._zeros.shape[0] < num_tracks:
            self._zeros = torch.zeros((max(num_tracks, 2 * self._zeros.shape[0]), 2), device=self.device)
        return self._zeros[:num_tracks]

    def _state(self, epoch):
        """The .state file's dict; the Social-NCE heads (which the .pkl predictor does not hold) under 'contrast'."""
        state = {'epoch': epoch, 'state_dict': self.model.state_dict(),
                 'optimizer': self.optimizer.state_dict(),
                 'scheduler': self.lr_scheduler.state_dict()}
        if self.contrast is not None:
            state['contrast'] = self.contrast.state_dict()
        return state

    def loop(self, train_scenes, val_scenes, train_goals, val_goals, out, epochs=35, start_epoch=0):
        for epoch in range(start_epoch, epochs):
            if epoch % self.save_every == 0:
                state = self._state(epoch)
                LSTMPredictor(self.model).save(state, out + '.epoch{}'.format(epoch))
            self.train(train_scenes, train_goals, epoch)
            if self.val_flag:
                self.val(val_scenes, val_goals, epoch)

        state = self._state(epoch + 1)
        LSTMPredictor(self.model).save(state, out + '.epoch{}'.format(epoch + 1))
        LSTMPredictor(self.model).save(state, out)

    def get_lr(self):
        for param_group in self.optimizer.param_groups:
            return param_group['lr']

    def train(self, scenes, goals, epoch):
        """One epoch over the SceneStore `scenes` (lstm/trainer.py:82-163)."""
        if goals is not None:
            raise NotImplementedError(GOALS_MESSAGE)
        start_time = time.time()

        print('epoch', epoch)
        plan = draw_epoch_plan(scenes.order, scenes.kept, self.batch_size, scenes.T, self.obs_length, self.augment,
                               self.augment_noise, self.obs_dropout)
        self.model.train()
        self.optimizer.zero_grad()

        gather_start = time.time()
        frame = scenes.frames(self.obs_length) if self.normalize_scene else None
        batches = scenes.gather(plan.order, self.batch_size, frame=frame, thetas=plan.thetas, noise=plan.noise,
                                noise_off=plan.noise_off)
        preprocess_time = time.time() - gather_start
        n = len(scenes)
        losses = []
        self._start_lengths = iter(plan.start_lengths) if plan.start_lengths is not None else None
        adv = self.adv_eps > 0
        nce = self.contrast is not None
        if adv:
            self._col_counts = torch.zeros(2, dtype=torch.float64, device=self.device)
        if nce:
            self._nce_losses = []
        try:
            for k, (batch_scene, batch_split) in enumerate(batches):
                batch_start = time.time()
                loss = self.train_batch(batch_scene, self._goals(batch_scene.shape[1]), torch.from_numpy(batch_split))
                losses.append(loss)
                last = min((k + 1) * self.batch_size, n)
                if last % (10 * self.batch_size) == 0:
                    loss_value = loss.item()
                    self.log.info({
                        'type': 'train',
                        'epoch': epoch, 'batch': last - 1, 'n_batches': n,
                        'time': round(time.time() - batch_start, 3),
                        'data_time': round(preprocess_time, 3),
                        'lr': self.get_lr(),
                        'loss': round(loss_value, 3),
                    })
            col = self._col_counts
            nce_losses = self._nce_losses
        finally:
            self._start_lengths = None
            self._col_counts = None
            self._nce_losses = None

        self.lr_scheduler.step()
        epoch_loss = 0.0
        values, nce_values = [], []
        if adv:               # the collision counts come back with the losses, in one copy
            values = torch.cat([torch.stack(losses).double(), col] if losses else [col]).cpu().tolist()
            values, col = values[:-2], values[-2:]
        elif nce:             # the L_nce values come back with the losses, in one copy
            values = torch.stack(losses + nce_losses).cpu().tolist() if losses else []
            values, nce_values = values[:len(losses)], values[len(losses):]
        elif losses:
            values = torch.stack(losses).cpu().tolist()
        for value in values:
            epoch_loss += value
        record = {
            'type': 'train-epoch',
            'epoch': epoch + 1,
            'loss': round(epoch_loss / (len(scenes)), 5),
            'time': round(time.time() - start_time, 1),
        }
        if adv:
            record['col_clean'] = col[0] / len(scenes)
            record['col_attacked'] = col[1] / len(scenes)
        if nce:
            record['loss_nce'] = round(sum(nce_values) / max(len(nce_values), 1), 5)
        self.log.info(record)

    def val(self, scenes, goals, epoch):
        """Validation over the SceneStore `scenes` in store order (lstm/trainer.py:165-227)."""
        if goals is not None:
            raise NotImplementedError(GOALS_MESSAGE)
        eval_start = time.time()
        self.model.train()
        frame = scenes.frames(self.obs_length) if self.normalize_scene else None
        losses, losses_test = [], []
        for batch_scene, batch_split in scenes.val_batches(self.batch_size, frame):
            loss, loss_test = self.val_batch(batch_scene, self._goals(batch_scene.shape[1]), torch.from_numpy(batch_split))
            losses.append(loss)
            losses_test.append(loss_test)
        values = torch.stack(losses + losses_test).cpu().tolist() if losses else []
        val_loss = 0.0
        test_loss = 0.0
        for v in values[:len(losses)]:
            val_loss += v
        for v in values[len(losses):]:
            test_loss += v
        eval_time = time.time() - eval_start

        self.log.info({
            'type': 'val-epoch',
            'epoch': epoch + 1,
            'loss': round(val_loss / (len(scenes)), 3),
            'test_loss': round(test_loss / len(scenes), 3),
            'time': round(eval_time, 1),
        })

    def train_batch(self, batch_scene, batch_scene_goal, batch_split):
        """lstm/trainer.py:229-269.  batch_scene [seq_length, num_tracks, 2], batch_split [batch_size + 1] (a host tensor
        keeps the layout lookups free of device syncs).  Returns the loss as a 0-dim device tensor."""
        if self.obs_dropout:
            self.start_length = (next(self._start_lengths) if self._start_lengths is not None
                                 else random.randint(0, self.obs_length - 2))

        observed = batch_scene[self.start_length:self.obs_length].clone()
        prediction_truth = batch_scene[self.obs_length:self.seq_length - 1].clone()
        targets = batch_scene[self.obs_length:self.seq_length] - batch_scene[self.obs_length - 1:self.seq_length - 1]

        def batch_loss(observed):
            rel_outputs, outputs = self.model(observed, batch_scene_goal, batch_split, prediction_truth)
            return task_loss(rel_outputs, outputs)

        def task_loss(rel_outputs, outputs):
            # For collision loss calculation
            primary_prediction = batch_scene[-self.pred_length:].clone()
            primary_prediction[:, batch_split[:-1]] = outputs[-self.pred_length:, batch_split[:-1]]

            ## Loss wrt primary tracks of each scene only
            return self.criterion(rel_outputs[-self.pred_length:], targets, batch_split,
                                  primary_prediction) * self.batch_size

        if self.adv_eps > 0:
            from ..attack import COL_LIMIT, pgd_collision
            res = pgd_collision(self.model, observed, batch_split, self.pred_length, self.adv_eps, self.adv_steps,
                                pad_to_batch_max=True)
            if self._col_counts is not None:
                self._col_counts += torch.stack([(res.d_clean <= COL_LIMIT).sum(), (res.d_best <= COL_LIMIT).sum()])
            if self.adv_wt < 1:
                loss = (1 - self.adv_wt) * batch_loss(observed) + self.adv_wt * batch_loss(res.observed)
            else:             # adv_wt = 1: the clean forward is not run
                loss = self.adv_wt * batch_loss(res.observed)
        elif self.contrast is not None:
            from .training import sequence_with_hidden
            rel_outputs, outputs, hidden = sequence_with_hidden(self.model, observed, batch_split, prediction_truth,
                                                                None)
            # the query: h of the step whose input was the last observed frame (observed starts at start_length)
            l_nce = self.contrast(batch_scene, hidden[observed.shape[0] - 2], batch_split, self.obs_length,
                                  layouts=self.model._layouts)
            loss = task_loss(rel_outputs, outputs) + self.contrast_weight * l_nce
            if self._nce_losses is not None:
                self._nce_losses.append(l_nce.detach())
        else:
            loss = batch_loss(observed)

        self.optimizer.zero_grad()
        loss.backward()
        self.optimizer.step()

        return loss.detach()

    def val_batch(self, batch_scene, batch_scene_goal, batch_split):
        """lstm/trainer.py:271-311: the teacher-forced and the free-running loss (model in train() mode, like the
        reference), as 0-dim device tensors."""
        if self.obs_dropout:
            self.start_length = 0

        observed = batch_scene[self.start_length:self.obs_length]
        prediction_truth = batch_scene[self.obs_length:self.seq_length - 1].clone()
        targets = batch_scene[self.obs_length:self.seq_length] - batch_scene[self.obs_length - 1:self.seq_length - 1]
        observed_test = observed.clone()

        with torch.no_grad():
            rel_outputs, _ = self.model(observed, batch_scene_goal, batch_split, prediction_truth)
            loss = self.criterion(rel_outputs[-self.pred_length:], targets, batch_split) * self.batch_size

            rel_outputs_test, _ = self.model(observed_test, batch_scene_goal, batch_split, n_predict=self.pred_length)
            loss_test = self.criterion(rel_outputs_test[-self.pred_length:], targets, batch_split) * self.batch_size

        return loss, loss_test


def prepare_data(path, subset='/train/', sample=1.0, goals=False, device=None):
    """lstm/data_load_utils.py:5-58 -> (SceneStore, None, True).  Files in os.listdir order, scenes in file order; a
    missing val folder gives (None, None, False), a missing train folder exits."""
    if goals:
        raise NotImplementedError(GOALS_MESSAGE)
    if not os.path.isdir(path + subset):
        if 'train' in subset:
            print("Train folder does NOT exist")
            sys.exit(1)
        if 'val' in subset:
            print("Validation folder does NOT exist")
            return None, None, False
    files = [f.split('.')[-2] for f in os.listdir(path + subset) if f.endswith('.ndjson')]
    store = SceneStore.from_files([path + subset + f + '.ndjson' for f in files], sample=sample, device=device)
    return store, None, True


class JsonLineFormatter(logging.Formatter):
    """One JSON object per record, with the fields of the reference's
    `jsonlogger.JsonFormatter('%(message)s %(levelname)s %(name)s %(asctime)s')`: a dict message is merged into the
    object (its `message` field is then null)."""

    def format(self, record):
        is_dict = isinstance(record.msg, dict)
        out = OrderedDict([('message', None if is_dict else record.getMessage()), ('levelname', record.levelname),
                           ('name', record.name), ('asctime', self.formatTime(record, self.datefmt))])
        if is_dict:
            out.update(record.msg)
        return json.dumps(out, default=str)


def build_parser(epochs=25):
    """The reference's flags (lstm/trainer.py:313-415)."""
    parser = argparse.ArgumentParser()
    parser.add_argument('--epochs', default=epochs, type=int,
                        help='number of epochs')
    parser.add_argument('--save_every', default=5, type=int,
                        help='frequency of saving model (in terms of epochs)')
    parser.add_argument('--obs_length', default=9, type=int,
                        help='observation length')
    parser.add_argument('--pred_length', default=12, type=int,
                        help='prediction length')
    parser.add_argument('--start_length', default=0, type=int,
                        help='starting time step of encoding observation')
    parser.add_argument('--batch_size', default=8, type=int)
    parser.add_argument('--lr', default=1e-3, type=float,
                        help='initial learning rate')
    parser.add_argument('--step_size', default=10, type=int,
                        help='step_size of lr scheduler')
    parser.add_argument('-o', '--output', default=None,
                        help='output file')
    parser.add_argument('--disable-cuda', action='store_true',
                        help='disable CUDA (refused: training runs on the GPU only)')
    parser.add_argument('--path', default='trajdata',
                        help='glob expression for data files')
    parser.add_argument('--goals', action='store_true',
                        help='flag to consider goals of pedestrians (refused: not built)')
    parser.add_argument('--loss', default='pred', choices=('L2', 'pred'),
                        help='loss objective, L2 loss (L2) and Gaussian loss (pred)')
    parser.add_argument('--type', default='vanilla',
                        choices=('vanilla', 'occupancy', 'directional', 'social', 'hiddenstatemlp',
                                 'nn', 'attentionmlp', 'nn_lstm', 'traj_pool'),
                        help='type of interaction encoder')
    parser.add_argument('--sample', default=1.0, type=float,
                        help='sample ratio when loading train/val scenes')
    parser.add_argument('--seed', type=int, default=42)

    ## Augmentations
    parser.add_argument('--augment', action='store_true',
                        help='perform rotation augmentation')
    parser.add_argument('--normalize_scene', action='store_true',
                        help='rotate scene so primary pedestrian moves northwards at end of observation')
    parser.add_argument('--augment_noise', action='store_true',
                        help='flag to add noise to observations for robustness')
    parser.add_argument('--obs_dropout', action='store_true',
                        help='perform observation length dropout')

    ## Loading pre-trained models
    pretrain = parser.add_argument_group('pretraining')
    pretrain.add_argument('--load-state', default=None,
                          help='load a pickled model state dictionary before training')
    pretrain.add_argument('--load-full-state', default=None,
                          help='load a pickled full state dictionary before training')
    pretrain.add_argument('--nonstrict-load-state', default=None,
                          help='load a pickled state dictionary before training')

    ## Sequence Encoder Hyperparameters
    hyperparameters = parser.add_argument_group('hyperparameters')
    hyperparameters.add_argument('--hidden-dim', type=int, default=128,
                                 help='LSTM hidden dimension')
    hyperparameters.add_argument('--coordinate-embedding-dim', type=int, default=64,
                                 help='coordinate embedding dimension')
    hyperparameters.add_argument('--pool_dim', type=int, default=256,
                                 help='output dimension of interaction vector')
    hyperparameters.add_argument('--goal_dim', type=int, default=64,
                                 help='goal embedding dimension')

    ## Grid-based pooling
    hyperparameters.add_argument('--cell_side', type=float, default=0.6,
                                 help='cell size of real world (in m) for grid-based pooling')
    hyperparameters.add_argument('--n', type=int, default=12,
                                 help='number of cells per side for grid-based pooling')
    hyperparameters.add_argument('--layer_dims', type=int, nargs='*', default=[512],
                                 help='interaction module layer dims for gridbased pooling')
    hyperparameters.add_argument('--embedding_arch', default='one_layer',
                                 help='interaction encoding arch for gridbased pooling')
    hyperparameters.add_argument('--pool_constant', default=0, type=int,
                                 help='background value (when cell empty) of gridbased pooling')
    hyperparameters.add_argument('--norm_pool', action='store_true',
                                 help='normalize the scene along direction of movement during grid-based pooling')
    hyperparameters.add_argument('--front', action='store_true',
                                 help='flag to only consider pedestrian in front during grid-based pooling')
    hyperparameters.add_argument('--latent_dim', type=int, default=16,
                                 help='latent dimension of encoding hidden dimension during social pooling')
    hyperparameters.add_argument('--norm', default=0, type=int,
                                 help='normalization scheme for input batch during grid-based pooling')

    ## Non-Grid-based pooling
    hyperparameters.add_argument('--no_vel', action='store_true',
                                 help='flag to not consider relative velocity of neighbours')
    hyperparameters.add_argument('--spatial_dim', type=int, default=32,
                                 help='embedding dimension for relative position')
    hyperparameters.add_argument('--vel_dim', type=int, default=32,
                                 help='embedding dimension for relative velocity')
    hyperparameters.add_argument('--neigh', default=4, type=int,
                                 help='number of nearest neighbours to consider')
    hyperparameters.add_argument('--mp_iters', default=5, type=int,
                                 help='message passing iterations in NMMP')

    ## Collision Loss
    hyperparameters.add_argument('--col_wt', default=0., type=float,
                                 help='collision loss weight')
    hyperparameters.add_argument('--col_distance', default=0.2, type=float,
                                 help='distance threshold post which collision occurs')

    ## Adversarial training against the collision attack (python -m trajnetplusplusbaselines_b200.attack)
    adversarial = parser.add_argument_group('adversarial training')
    adversarial.add_argument('--adv_eps', default=0., type=float,
                             help='radius (m) of the per-frame L2 ball the primary\'s observation is attacked in; '
                                  '0 trains without the attack')
    adversarial.add_argument('--adv_steps', default=5, type=int,
                             help='PGD iterations of the attack per training batch')
    adversarial.add_argument('--adv_wt', default=0.5, type=float,
                             help='weight of the attacked loss, in (0, 1]; the clean loss gets 1 - adv_wt')

    ## Social-NCE contrastive term (lstm/contrast.py)
    contrast = parser.add_argument_group('social-nce')
    contrast.add_argument('--contrast_weight', default=0., type=float,
                          help='weight of the Social-NCE term added to the training loss; 0 trains without it')
    contrast.add_argument('--contrast_horizon', default=4, type=int,
                          help='future steps whose positions make the Social-NCE samples, in [1, pred_length]')
    contrast.add_argument('--contrast_temperature', default=0.1, type=float,
                          help='temperature of the Social-NCE softmax, > 0')
    return parser


def build_model(args):
    """The interaction module and the LSTM as the reference CLI builds them (lstm/trainer.py:465-494)."""
    pool = None
    if args.type == 'hiddenstatemlp':
        pool = HiddenStateMLPPooling(hidden_dim=args.hidden_dim, out_dim=args.pool_dim,
                                     mlp_dim_vel=args.vel_dim)
    elif args.type == 'attentionmlp':
        pool = AttentionMLPPooling(hidden_dim=args.hidden_dim, out_dim=args.pool_dim,
                                   mlp_dim_spatial=args.spatial_dim, mlp_dim_vel=args.vel_dim)
    elif args.type == 'nn':
        pool = NearestNeighborMLP(n=args.neigh, out_dim=args.pool_dim, no_vel=args.no_vel)
    elif args.type == 'nn_lstm':
        pool = NearestNeighborLSTM(n=args.neigh, hidden_dim=args.hidden_dim, out_dim=args.pool_dim)
    elif args.type == 'traj_pool':
        pool = TrajectronPooling(hidden_dim=args.hidden_dim, out_dim=args.pool_dim)
    elif args.type != 'vanilla':
        pool = GridBasedPooling(type_=args.type, hidden_dim=args.hidden_dim,
                                cell_side=args.cell_side, n=args.n, front=args.front,
                                out_dim=args.pool_dim, embedding_arch=args.embedding_arch,
                                constant=args.pool_constant, pretrained_pool_encoder=None,
                                norm=args.norm, layer_dims=args.layer_dims, latent_dim=args.latent_dim)
    return LSTM(pool=pool,
                embedding_dim=args.coordinate_embedding_dim,
                hidden_dim=args.hidden_dim,
                goal_flag=args.goals,
                goal_dim=args.goal_dim)


def main(argv=None, epochs=25):
    """`python -m trajnetplusplusbaselines_b200.lstm.trainer`: the reference's CLI (lstm/trainer.py:313-531), on CUDA.
    Reads DATA_BLOCK/<path>/{train,val}/*.ndjson, writes OUTPUT_BLOCK/<path>/lstm_<type>_<output>.pkl (+ .epoch<k>,
    .state, .log) relative to the working directory."""
    parser = build_parser(epochs)
    args = parser.parse_args(argv)
    if args.disable_cuda:
        sys.exit("--disable-cuda: there is no CPU path, training runs on the GPU")
    if not args.adv_eps >= 0:
        sys.exit("--adv_eps must be >= 0 (got %g)" % args.adv_eps)
    if args.adv_steps < 1:
        sys.exit("--adv_steps must be >= 1 (got %d)" % args.adv_steps)
    if not 0 < args.adv_wt <= 1:
        sys.exit("--adv_wt must be in (0, 1] (got %g)" % args.adv_wt)
    if not args.contrast_weight >= 0:
        sys.exit("--contrast_weight must be >= 0 (got %g)" % args.contrast_weight)
    if args.contrast_weight > 0:          # the term's other flags matter only when it is on
        if not 1 <= args.contrast_horizon <= args.pred_length:
            sys.exit("--contrast_horizon must be in [1, pred_length = %d] (got %d)"
                     % (args.pred_length, args.contrast_horizon))
        if not args.contrast_temperature > 0:
            sys.exit("--contrast_temperature must be > 0 (got %g)" % args.contrast_temperature)
        if args.adv_eps > 0:
            sys.exit("--contrast_weight > 0 together with --adv_eps > 0 is not built")

    ## Set seed for reproducibility
    torch.manual_seed(args.seed)
    random.seed(args.seed)

    # the model first (torch's generator only; data loading draws from none but `random`, and only at --sample < 1):
    # a configuration the training backward does not support is refused before any file is touched
    try:
        model = build_model(args)
        check_trainable(model)
        if args.adv_eps > 0:
            from .training import check_rollout
            check_rollout(model)
        contrast = None
        if args.contrast_weight > 0:      # after the model: its initialisation draws what a run without the term draws
            from .contrast import SocialNCE, check_contrast
            check_contrast(model)
            contrast = SocialNCE(model.hidden_dim, horizon=args.contrast_horizon,
                                 temperature=args.contrast_temperature)
    except (NotImplementedError, RuntimeError, ValueError) as e:
        sys.exit(str(e))

    ## Define location to save trained model
    if not os.path.exists('OUTPUT_BLOCK/{}'.format(args.path)):
        os.makedirs('OUTPUT_BLOCK/{}'.format(args.path))
    args.output = 'OUTPUT_BLOCK/{}/lstm_{}_{}.pkl'.format(args.path, args.type, args.output)

    # configure logging: JSON lines to <output>.log, the records' text to stdout
    file_handler = logging.FileHandler(args.output + '.log', mode='a' if args.load_full_state else 'w')
    file_handler.setFormatter(JsonLineFormatter())
    stdout_handler = logging.StreamHandler(sys.stdout)
    root = logging.getLogger()
    old_level = root.level
    root.setLevel(logging.INFO)
    root.addHandler(stdout_handler)
    root.addHandler(file_handler)
    try:
        logging.info({
            'type': 'process',
            'argv': sys.argv if argv is None else [sys.argv[0]] + list(argv),
            'args': vars(args),
            'version': int(_lib.load().tb2_version()),
            'hostname': socket.gethostname(),
        })

        # refactor args for --load-state
        args.load_state_strict = True
        if args.nonstrict_load_state:
            args.load_state = args.nonstrict_load_state
            args.load_state_strict = False
        if args.load_full_state:
            args.load_state = args.load_full_state

        _lib.require_cuda()
        args.device = torch.device('cuda', torch.cuda.current_device())

        args.path = 'DATA_BLOCK/' + args.path
        ## Prepare data
        train_scenes, train_goals, _ = prepare_data(args.path, subset='/train/', sample=args.sample, device=args.device)
        val_scenes, val_goals, val_flag = prepare_data(args.path, subset='/val/', sample=args.sample, device=args.device)

        model = model.to(args.device)
        optimizer = torch.optim.Adam(model.parameters(), lr=args.lr, weight_decay=1e-4)
        if contrast is not None:          # the heads' group, before the scheduler records each group's lr
            contrast = contrast.to(args.device)
            optimizer.add_param_group({'params': list(contrast.parameters())})
        lr_scheduler = None
        if args.step_size is not None:
            lr_scheduler = torch.optim.lr_scheduler.StepLR(optimizer, args.step_size)
        start_epoch = 0

        # Loss Criterion
        criterion = L2Loss(col_wt=args.col_wt, col_distance=args.col_distance) if args.loss == 'L2' \
            else PredictionLoss(col_wt=args.col_wt, col_distance=args.col_distance)

        if args.load_state:
            print("Loading Model Dict")
            with open(args.load_state, 'rb') as f:
                checkpoint = torch.load(f, map_location=args.device)
            # a full state's optimizer has one parameter group more with the Social-NCE heads: resume like with like
            if args.load_full_state and contrast is not None and 'contrast' not in checkpoint:
                sys.exit("%s holds no Social-NCE heads: it was not trained with --contrast_weight > 0" % args.load_state)
            if args.load_full_state and contrast is None and 'contrast' in checkpoint:
                sys.exit("%s holds Social-NCE heads: resume it with --contrast_weight > 0" % args.load_state)
            model.load_state_dict(checkpoint['state_dict'], strict=args.load_state_strict)
            if args.load_full_state and contrast is not None:
                contrast.load_state_dict(checkpoint['contrast'])
            if args.load_full_state:
                print("Loading Optimizer Dict")
                optimizer.load_state_dict(checkpoint['optimizer'])
                lr_scheduler.load_state_dict(checkpoint['scheduler'])
                start_epoch = checkpoint['epoch']

        trainer = Trainer(model, optimizer=optimizer, lr_scheduler=lr_scheduler, device=args.device,
                          criterion=criterion, batch_size=args.batch_size, obs_length=args.obs_length,
                          pred_length=args.pred_length, augment=args.augment, normalize_scene=args.normalize_scene,
                          save_every=args.save_every, start_length=args.start_length, obs_dropout=args.obs_dropout,
                          augment_noise=args.augment_noise, val_flag=val_flag, adv_eps=args.adv_eps,
                          adv_steps=args.adv_steps, adv_wt=args.adv_wt, contrast_weight=args.contrast_weight,
                          contrast=contrast)
        trainer.loop(train_scenes, val_scenes, train_goals, val_goals, args.output, epochs=args.epochs,
                     start_epoch=start_epoch)
    finally:
        root.removeHandler(stdout_handler)
        root.removeHandler(file_handler)
        file_handler.close()
        root.setLevel(old_level)


if __name__ == '__main__':
    main()
