"""
Trainers for semantic segmentation and image<->spectrum models with the reference's public
surface (atomai/trainers/trainer.py:42-857): BaseTrainer / SegTrainer / ImSpecTrainer, same method
names, keyword arguments, training-loop semantics ("one cycle = one train mini-batch + one test
mini-batch" unless full_epoch), loss histories and checkpoint dictionary.

What is different underneath:
  * `self.net(feat)`, `self.criterion(...)`, `loss.backward()` and `optimizer.step()` — the seam
    into the hot path, trainer.py:204-207 — run as hand-written sm_90a kernels (native tape,
    fused loss, fused multi-tensor Adam);
  * data parallelism over the GPUs of one box when launched under torchrun: mini-batches are
    sharded along N, gradients all-reduced once per step over NCCL (atomai_b200/parallel.py).
"""
import copy
import warnings
from collections import OrderedDict
from typing import Callable, Dict, List, Optional, Tuple, Type, Union

import numpy as np
import torch

from .. import losses_metrics
from ..nets import init_fcnn_model
from ..optim import FusedAdam
from ..parallel import Comm, GradBucket, broadcast_model
from ..utils.nn import (average_weights, gpu_usage_map, reset_bnorm, set_train_rng,
                        weights_init)
from ..utils.preproc import (array2list, init_dataloaders, init_fcnn_dataloaders,
                             init_imspec_dataloaders, preprocess_training_image_data,
                             preprocess_training_imspec_data, shard_batches)

augfn_type = Callable[[torch.Tensor, torch.Tensor, int], Tuple[torch.Tensor, torch.Tensor]]


def _shuffle(idx: np.ndarray, seed: int) -> np.ndarray:
    """sklearn.utils.shuffle(idx, random_state=seed) — same permutation, without the import cost."""
    try:
        from sklearn.utils import shuffle
        return shuffle(idx, random_state=seed)
    except Exception:  # noqa
        return np.random.RandomState(seed).permutation(idx)


class BaseTrainer:
    """
    Base trainer class for training semantic segmentation and image-to-spectrum /
    spectrum-to-image deep learning models (API of atomai/trainers/trainer.py:42-607).

    Example:

    >>> t = BaseTrainer()
    >>> t.set_model(atomai_b200.nets.Unet(), nb_classes=1)
    >>> t.compile_trainer((images, labels, images_test, labels_test),
    >>>                   loss="ce", full_epoch=True, training_cycles=25, swa=True)
    >>> t.fit()
    >>> t.save_model("my_model")
    """
    def __init__(self):
        set_train_rng(1)
        self.device = 'cuda' if torch.cuda.is_available() else 'cpu'
        self.net = None
        self.criterion = None
        self.optimizer = None
        self.compute_accuracy = False
        self.full_epoch = True
        self.swa = False
        self.perturb_weights = False
        self.running_weights = {}
        self.training_cycles = 0
        self.batch_idx_train, self.batch_idx_test = [], []
        self.batch_size = 1
        self.nb_classes = None
        self.X_train, self.y_train = None, None
        self.X_test, self.y_test = None, None
        self.train_loader = torch.utils.data.TensorDataset()
        self.test_loader = torch.utils.data.TensorDataset()
        self.data_is_set = False
        self.augdict = {}
        self.augment_fn = None
        self.filename = "model"
        self.print_loss = 1
        self.meta_state_dict = dict()
        self.loss_acc = {"train_loss": [], "test_loss": [],
                         "train_accuracy": [], "test_accuracy": []}
        self.lr_scheduler = None
        self.accuracy_metrics = None
        self.plot_training_history = True
        # data parallelism (new): filled by compile_trainer when torch.distributed is initialised
        self.comm: Optional[Comm] = None
        self._bucket: Optional[GradBucket] = None
        self.sync_host = True     # loss.item() every step like the reference (trainer.py:210)

    # ------------------------------------------------------------------ small helpers
    def _reset_rng(self, seed: int) -> None:
        set_train_rng(seed)

    def _reset_weights(self) -> None:
        """Xavier re-initialisation of conv/linear layers + BatchNorm reset."""
        self.net.apply(weights_init)
        self.net.apply(reset_bnorm)

    def _reset_training_history(self) -> None:
        self.loss_acc = {"train_loss": [], "test_loss": [],
                         "train_accuracy": [], "test_accuracy": []}

    def _delete_optimizer(self) -> None:
        self.optimizer = None

    @property
    def _world(self) -> int:
        return self.comm.world if self.comm is not None else 1

    def _is_main(self) -> bool:
        if self.comm is not None:
            return self.comm.rank == 0
        d = torch.distributed
        return not (d.is_available() and d.is_initialized()) or d.get_rank() == 0

    # ------------------------------------------------------------------ data / model
    def set_data(self, X_train, y_train, X_test, y_test, **kwargs: float) -> None:
        """
        Sets training and test data: DataLoaders (full_epoch) or lists of batch tensors from which
        one element is taken per training cycle (atomai/trainers/trainer.py:129-162).
        """
        memory_alloc = kwargs.get("memory_alloc", 4)
        tor = lambda x: torch.from_numpy(x) if isinstance(x, np.ndarray) else x  # noqa: E731
        X_train, y_train, X_test, y_test = tor(X_train), tor(y_train), tor(X_test), tor(y_test)
        if self.full_epoch:
            self.train_loader, self.test_loader = init_dataloaders(
                X_train, y_train, X_test, y_test, self.batch_size, memory_alloc)
        else:
            (self.X_train, self.y_train, self.X_test, self.y_test) = array2list(
                X_train, y_train, X_test, y_test, self.batch_size, memory_alloc)
        self.data_is_set = True

    def set_model(self, model: Type[torch.nn.Module], nb_classes: int = None) -> None:
        self.net = model
        self.net.to(self.device)
        if self.nb_classes is None and nb_classes:
            self.nb_classes = nb_classes

    def get_loss_fn(self, loss: Union[str, Callable] = 'mse', nb_classes: int = None):
        """'mse', 'ce' or a custom callable (atomai/trainers/trainer.py:178-187)."""
        return losses_metrics.select_loss(loss, nb_classes)

    # ------------------------------------------------------------------ the hot loop
    def _require_cuda(self) -> None:
        if self.device != 'cuda':
            raise RuntimeError(
                "atomai_b200 trains on CUDA (H100, sm_90a) only: the native kernels have no CPU "
                "fallback. Use the reference AtomAI for CPU training.")

    def train_step(self, feat: torch.Tensor, tar: torch.Tensor) -> Tuple[float]:
        """
        Forward, loss, backward, optimizer step on one mini-batch
        (atomai/trainers/trainer.py:189-211).
        """
        self._require_cuda()
        self.net.train()
        self.optimizer.zero_grad(set_to_none=self._bucket is None)
        if self._bucket is not None:
            self._bucket.zero_()
        feat, tar = feat.to(self.device), tar.to(self.device)
        prob = self.net(feat)
        loss = self.criterion(prob, tar)
        loss.backward()
        if self._bucket is not None:
            self._bucket.attach()
            self._bucket.allreduce(self.comm)
        self.optimizer.step()
        if self.comm is not None and self.comm.world > 1:
            loss = loss.detach().clone()
            self.comm.allreduce_any_(loss)
            loss = loss / self.comm.world
        if self.compute_accuracy:
            acc_score = self.accuracy_fn(tar, prob)
            return (loss.item() if self.sync_host else loss.detach(), acc_score)
        return (loss.item() if self.sync_host else loss.detach(),)

    def test_step(self, feat: torch.Tensor, tar: torch.Tensor) -> float:
        """Forward pass on test data without autograd (atomai/trainers/trainer.py:213-231)."""
        self._require_cuda()
        feat, tar = feat.to(self.device), tar.to(self.device)
        self.net.eval()
        with torch.no_grad():
            prob = self.net(feat)
            loss = self.criterion(prob, tar)
        if self.comm is not None and self.comm.world > 1:
            loss = loss.detach().clone()
            self.comm.allreduce_any_(loss)
            loss = loss / self.comm.world
        if self.compute_accuracy:
            acc_score = self.accuracy_fn(tar, prob)
            return (loss.item() if self.sync_host else loss.detach(), acc_score)
        return (loss.item() if self.sync_host else loss.detach(),)

    def _issue_batches(self, e: int):
        """The four tensors of cycle `e` on the device.  Host-resident (pinned) batches — data sets
        larger than `memory_alloc`, the reference keeps those on the CPU too
        (atomai/utils/preproc.py:170-201) — are copied on a side stream so that the transfer of
        cycle e+1 overlaps the kernels of cycle e; returns (tensors, event or None)."""
        f, t = self.dataloader(self.batch_idx_train[e], mode='train')
        # the reference fetches the test batch after appending the train loss, i.e. its
        # augmentation seed is one higher (atomai/trainers/trainer.py:239-246)
        f_, t_ = self.dataloader(self.batch_idx_test[e], mode='test', _seed_offset=1)
        host = [x for x in (f, t, f_, t_) if isinstance(x, torch.Tensor) and not x.is_cuda]
        if not host or self.device != 'cuda':
            return (f, t, f_, t_), None
        if getattr(self, "_copy_stream", None) is None:
            self._copy_stream = torch.cuda.Stream()
        with torch.cuda.stream(self._copy_stream):
            dev = tuple(x.to(self.device, non_blocking=True) for x in (f, t, f_, t_))
            ev = torch.cuda.Event()
            ev.record(self._copy_stream)
        return dev, ev

    def step(self, e: int) -> None:
        """One train mini-batch + one test mini-batch (atomai/trainers/trainer.py:233-251)."""
        pre = getattr(self, "_prefetched", None)
        if pre is not None and pre[0] == e:
            batches, ev = pre[1]
        else:
            batches, ev = self._issue_batches(e)
        self._prefetched = None
        if ev is not None:
            cur = torch.cuda.current_stream()
            cur.wait_event(ev)
            for x in batches:
                x.record_stream(cur)
            if e + 1 < len(self.batch_idx_train) and self.augment_fn is None:
                self._prefetched = (e + 1, self._issue_batches(e + 1))
        features, targets, features_, targets_ = batches
        loss = self.train_step(features, targets)
        self.loss_acc["train_loss"].append(loss[0])
        loss_ = self.test_step(features_, targets_)
        self.loss_acc["test_loss"].append(loss_[0])
        if self.compute_accuracy:
            self.loss_acc["train_accuracy"].append(loss[1])
            self.loss_acc["test_accuracy"].append(loss_[1])

    def step_full(self) -> None:
        """All mini-batches once (atomai/trainers/trainer.py:253-287)."""
        c, c_test = 0, 0
        losses, losses_test = 0, 0
        acc, acc_test = 0, 0
        for features, targets in self.train_loader:
            features, targets = self._shard(features, targets)
            if self.augment_fn is not None:
                features, targets = self.augment_fn(features, targets, seed=c)
            loss = self.train_step(features, targets)
            losses += loss[0]
            if self.compute_accuracy:
                acc += loss[1]
            c += 1
        for features_, targets_ in self.test_loader:
            features_, targets_ = self._shard(features_, targets_)
            if self.augment_fn is not None:
                features_, targets_ = self.augment_fn(features_, targets_, seed=c_test)
            loss_ = self.test_step(features_, targets_)
            losses_test += loss_[0]
            if self.compute_accuracy:
                acc_test += loss_[1]
            c_test += 1
        self.loss_acc["train_loss"].append(losses / c)
        self.loss_acc["test_loss"].append(losses_test / c_test)
        if self.compute_accuracy:
            self.loss_acc["train_accuracy"].append(acc / c)
            self.loss_acc["test_accuracy"].append(acc_test / c_test)

    def _shard(self, x: torch.Tensor, y: torch.Tensor):
        if self._world == 1:
            return x, y
        k = x.shape[0] // self._world
        r = self.comm.rank
        return x[r * k:(r + 1) * k], y[r * k:(r + 1) * k]

    def eval_model(self) -> None:
        """Evaluates the model on the entire test set (atomai/trainers/trainer.py:289-324)."""
        self.net.eval()
        running_loss_test, running_acc_test, c = 0, 0, 0
        if self.full_epoch:
            for features_, targets_ in self.test_loader:
                features_, targets_ = self._shard(features_, targets_)
                loss_ = self.test_step(features_, targets_)
                running_loss_test += float(loss_[0])
                if self.compute_accuracy:
                    running_acc_test += float(loss_[1])
                c += 1
        else:
            for idx in range(len(self.X_test)):
                features_, targets_ = self.dataloader(idx, mode='test')
                loss_ = self.test_step(features_, targets_)
                running_loss_test += float(loss_[0])
                if self.compute_accuracy:
                    running_acc_test += float(loss_[1])
            c = len(self.X_test)
        if self._is_main():
            print('Model (final state) evaluation loss:', np.around(running_loss_test / c, 4))
            if self.compute_accuracy:
                print('Model (final state) accuracy:', np.around(running_acc_test / c, 4))

    def dataloader(self, batch_num: int, mode: str = 'train', _seed_offset: int = 0) -> Tuple[torch.Tensor]:
        """Picks one pre-chunked batch (atomai/trainers/trainer.py:326-342)."""
        if mode == 'test':
            features = self.X_test[batch_num][:self.batch_size]
            targets = self.y_test[batch_num][:self.batch_size]
        else:
            features = self.X_train[batch_num][:self.batch_size]
            targets = self.y_train[batch_num][:self.batch_size]
        if self.augment_fn is not None:
            features, targets = self.augment_fn(
                features, targets, seed=len(self.loss_acc["train_loss"]) + _seed_offset)
        return features, targets

    # ------------------------------------------------------------------ bookkeeping
    def save_model(self, *args: str) -> None:
        """
        Saves weights, optimizer and architecture meta-data as `<filename>.tar`
        (checkpoint dictionary of atomai/trainers/trainer.py:344-358; rank 0 only).
        """
        filename = args[0] if len(args) > 0 else self.filename
        self.meta_state_dict["weights"] = self.meta_state_dict.get(
            "weights", self.net.state_dict())
        self.meta_state_dict["optimizer"] = self.meta_state_dict.get(
            "optimizer", self.optimizer)
        if self._is_main():
            torch.save(self.meta_state_dict, filename + '.tar')

    def print_statistics(self, e: int, **kwargs) -> None:
        """Loss / accuracy / GPU memory line (atomai/trainers/trainer.py:360-395)."""
        if not self._is_main():
            return
        accuracy_metrics = self.accuracy_metrics or "Accuracy"
        if torch.cuda.is_available():
            gpu_usage = gpu_usage_map(torch.cuda.current_device())
        else:
            gpu_usage = ['N/A ', ' N/A']
        msg = ['Epoch {}/{} ...'.format(e + 1, self.training_cycles),
               'Training loss: {} ...'.format(np.around(float(self.loss_acc["train_loss"][-1]), 4)),
               'Test loss: {} ...'.format(np.around(float(self.loss_acc["test_loss"][-1]), 4))]
        if self.compute_accuracy:
            msg += ['Train {}: {} ...'.format(
                        accuracy_metrics, np.around(float(self.loss_acc["train_accuracy"][-1]), 4)),
                    'Test {}: {} ...'.format(
                        accuracy_metrics, np.around(float(self.loss_acc["test_accuracy"][-1]), 4))]
        msg.append('GPU memory usage: {}/{}'.format(gpu_usage[0], gpu_usage[1]))
        print(*msg)

    def accuracy_fn(self, *args) -> None:
        raise NotImplementedError

    def weight_perturbation(self, e: int) -> None:
        """Time-dependent weight perturbation w <- w + N(0, a/(1+e)^gamma)
        (atomai/trainers/trainer.py:403-416)."""
        a = self.perturb_weights["a"]
        gamma = self.perturb_weights["gamma"]
        e_p = self.perturb_weights["e_p"]
        if self.perturb_weights and (e + 1) % e_p == 0:
            var = torch.tensor(a / (1 + e)**gamma)
            sd = self.net.state_dict()
            for k, v in sd.items():
                if v.dtype.is_floating_point:
                    v.add_(torch.randn_like(v) * torch.sqrt(var))

    def save_running_weights(self, e: int) -> None:
        """Keeps the last 30 (5 for full_epoch) state_dicts on the CPU for SWA
        (atomai/trainers/trainer.py:418-429)."""
        swa_epochs = 5 if self.full_epoch else 30
        if self.training_cycles - e <= swa_epochs:
            i_ = swa_epochs - (self.training_cycles - e)
            self.running_weights[i_] = OrderedDict(
                (k, v.detach().clone().cpu()) for k, v in self.net.state_dict().items())

    def data_augmentation(self, augment_fn: augfn_type) -> None:
        self.augment_fn = augment_fn

    def compile_trainer(self,
                        train_data=None,
                        loss: Union[str, Callable] = 'ce',
                        optimizer: Optional[Type[torch.optim.Optimizer]] = None,
                        training_cycles: int = 1000,
                        batch_size: int = 32,
                        compute_accuracy: bool = False,
                        full_epoch: bool = False,
                        swa: bool = False,
                        perturb_weights: bool = False,
                        **kwargs):
        """
        Compile a trainer — arguments and kwargs (lr_scheduler, batch_seed,
        overwrite_train_data, memory_alloc, print_loss, accuracy_metrics, filename,
        plot_training_history) as in atomai/trainers/trainer.py:441-565.  New optional kwargs:
        sync_bn (bool, default True) for data-parallel runs, sync_host (bool, default True:
        read the loss back every step like the reference).
        """
        self.full_epoch = full_epoch
        self.training_cycles = training_cycles
        self.batch_size = batch_size
        self.compute_accuracy = compute_accuracy
        self.swa = swa
        self.lr_scheduler = kwargs.get("lr_scheduler")
        self.sync_host = kwargs.get("sync_host", True)
        alloc = kwargs.get("memory_alloc", 4)

        if torch.distributed.is_available() and torch.distributed.is_initialized() \
                and torch.distributed.get_world_size() > 1 and not getattr(self, "_no_dp", False):
            self.comm = Comm(sync_bn=kwargs.get("sync_bn", True))
            if batch_size % self.comm.world != 0:
                raise ValueError(f"batch_size={batch_size} must be divisible by the number of "
                                 f"data-parallel ranks ({self.comm.world})")

        data_was_set = False
        if not self.data_is_set or kwargs.get("overwrite_train_data", True):
            self.set_data(*train_data, memory_alloc=alloc)
            data_was_set = True
        if self.comm is not None and not self.full_epoch and not data_was_set:
            self.batch_size = batch_size // self.comm.world      # batches are already sharded
        if self.comm is not None and not self.full_epoch and data_was_set:
            r, w = self.comm.rank, self.comm.world
            self.X_train, self.y_train = shard_batches(self.X_train, r, w), shard_batches(self.y_train, r, w)
            self.X_test, self.y_test = shard_batches(self.X_test, r, w), shard_batches(self.y_test, r, w)
            self.batch_size = batch_size // w

        self.perturb_weights = perturb_weights
        if self.perturb_weights:
            if self.meta_state_dict.get("batch_norm", self.meta_state_dict.get("batchnorm")):
                raise AssertionError(
                    "To use time-dependent weights perturbation, " +
                    "turn off the batch normalization layes")
            if isinstance(self.perturb_weights, bool):
                e_p = 1 if self.full_epoch else 50
                self.perturb_weights = {"a": .01, "gamma": 1.5, "e_p": e_p}

        if self.comm is not None:
            broadcast_model(self.net, self.comm)
            self.net._comm = self.comm
        params = list(self.net.parameters())
        if self.optimizer is None:
            if optimizer is None:
                if self.device == 'cuda':
                    self.optimizer = FusedAdam(params, lr=1e-3)
                else:   # structural / CPU-side use only; training itself requires CUDA
                    self.optimizer = torch.optim.Adam(params, lr=1e-3)
            else:
                self.optimizer = optimizer(params)
        if self.comm is not None:
            self._bucket = GradBucket(params)
            # 1/world averaging: folded into the fused Adam kernel, or applied to the bucket for
            # any other (user-supplied) optimizer
            if isinstance(self.optimizer, FusedAdam):
                self.optimizer.grad_scale = 1.0 / self.comm.world
                self._bucket.post_scale = 1.0
            else:
                self._bucket.post_scale = 1.0 / self.comm.world
        if self.criterion is None:
            self.criterion = self.get_loss_fn(loss, self.nb_classes)
        if self.comm is not None and isinstance(self.criterion, (losses_metrics.dice_loss,
                                                                 losses_metrics.focal_loss)):
            # not per-pixel means: the loss adds its sums over the ranks before it finalises
            self.criterion.comm = self.comm

        if not self.full_epoch:
            seed = kwargs.get("batch_seed", 1)
            r = self.training_cycles // len(self.X_train)
            idx_tr = np.arange(len(self.X_train)).repeat(r + 1)[:self.training_cycles]
            r_ = self.training_cycles // len(self.X_test)
            idx_te = np.arange(len(self.X_test)).repeat(r_ + 1)[:self.training_cycles]
            self.batch_idx_train = _shuffle(idx_tr, seed)
            self.batch_idx_test = _shuffle(idx_te, seed)

        self.print_loss = kwargs.get("print_loss")
        if self.print_loss is None:
            self.print_loss = 1 if self.full_epoch else 100
        self.accuracy_metrics = kwargs.get("accuracy_metrics")
        self.filename = kwargs.get("filename", "./model")
        self.plot_training_history = kwargs.get("plot_training_history", True)

    def select_lr(self, e: int) -> None:
        lr_i = self.lr_scheduler[e] if e < len(self.lr_scheduler) else self.lr_scheduler[-1]
        for g in self.optimizer.param_groups:
            g['lr'] = lr_i

    def run(self) -> Type[torch.nn.Module]:
        """
        Trains the network, prints statistics, saves the final checkpoint
        (atomai/trainers/trainer.py:573-604).
        """
        for e in range(self.training_cycles):
            if self.lr_scheduler is not None:
                self.select_lr(e)
            if self.full_epoch:
                self.step_full()
            else:
                self.step(e)
            if self.swa:
                self.save_running_weights(e)
            if self.perturb_weights:
                self.weight_perturbation(e)
            if any([e == 0, (e + 1) % self.print_loss == 0, e == self.training_cycles - 1]):
                self.print_statistics(e)
        if not self.sync_host:   # deferred read-back: one sync at the end instead of one per step
            for k in ("train_loss", "test_loss", "train_accuracy", "test_accuracy"):
                self.loss_acc[k] = [float(v) for v in self.loss_acc[k]]
        if not self.full_epoch:
            self.eval_model()
        if self.swa:
            if self._is_main():
                print("Performing stochastic weight averaging...")
            self.net.load_state_dict(average_weights(self.running_weights))
            self.eval_model()
        self.save_model(self.filename + "_metadict_final")
        if self.plot_training_history and self._is_main():
            try:
                from ..utils.viz import plot_losses
                plot_losses(self.loss_acc["train_loss"], self.loss_acc["test_loss"])
            except Exception:  # noqa  (matplotlib is optional)
                pass
        return self.net

    def fit(self) -> None:
        _ = self.run()


class SegTrainer(BaseTrainer):
    """
    Class for training a fully convolutional neural network for semantic segmentation of noisy
    experimental data.  Arguments as in atomai/trainers/trainer.py:610-671: `model` ('Unet',
    'dilnet' or a custom fully convolutional torch module), `nb_classes`, and the kwargs
    seed, batch_seed, batch_norm, dropout, upsampling, nb_filters, with_dilation, layers.
    """
    def __init__(self,
                 model: Union[Type[torch.nn.Module], str] = "Unet",
                 nb_classes: int = 1,
                 **kwargs: Union[int, List, str, bool]) -> None:
        super(SegTrainer, self).__init__()
        seed = kwargs.get("seed", 1)
        kwargs["batch_seed"] = kwargs.get("batch_seed", seed)
        set_train_rng(seed)
        self.nb_classes = nb_classes
        self.net, self.meta_state_dict = init_fcnn_model(model, self.nb_classes, **kwargs)
        self.net.to(self.device)
        if self.device == 'cpu':
            warnings.warn("No GPU found. atomai_b200 cannot train without an H100 (sm_90a)",
                          UserWarning)
        self.meta_state_dict["weights"] = self.net.state_dict()

    def set_data(self, X_train, y_train, X_test=None, y_test=None,
                 **kwargs: Union[float, int]) -> None:
        """
        Sets training and test data (atomai/trainers/trainer.py:673-730): images
        (n, 1, h, w) or (n, h, w); masks (n, 1, h, w) binary / (n, h, w) multiclass; an optional
        train/test split (test_size, seed) when no test set is given; memory_alloc.
        """
        if X_test is None or y_test is None:
            from sklearn.model_selection import train_test_split
            X_train, X_test, y_train, y_test = train_test_split(
                X_train, y_train, test_size=kwargs.get("test_size", .15),
                shuffle=True, random_state=kwargs.get("seed", 1))
        if self.full_epoch:
            self.train_loader, self.test_loader, nb_classes = init_fcnn_dataloaders(
                X_train, y_train, X_test, y_test, self.batch_size,
                memory_alloc=kwargs.get("memory_alloc", 4))
        else:
            (self.X_train, self.y_train, self.X_test, self.y_test,
             nb_classes) = preprocess_training_image_data(
                 X_train, y_train, X_test, y_test, self.batch_size, kwargs.get("memory_alloc", 4))
        self.data_is_set = True
        if self.nb_classes != nb_classes:
            raise AssertionError("Number of classes in initialized model" +
                                 " is different from the number of classes" +
                                 " contained in training data")

    def accuracy_fn(self, y: torch.Tensor, y_prob: torch.Tensor, *args):
        """Mean IoU of the batch (atomai/trainers/trainer.py:731-737), counted on the GPU; a float
        per step, or a device scalar read back at the end of the run with sync_host=False.  Under
        data parallelism the confusion counts are added over the ranks first."""
        iou = losses_metrics.IoU(y, y_prob, self.nb_classes,
                                 comm=self.comm if self._world > 1 else None)
        return iou.evaluate() if self.sync_host else iou.evaluate_device()


class ImSpecTrainer(BaseTrainer):
    """
    Trainer of an encoder-decoder model mapping images to spectra or spectra to images
    (atomai/trainers/trainer.py:740-857): in_dim, out_dim, latent_dim and the kwargs seed,
    batch_seed, nblayers_encoder, nblayers_decoder, nbfilters_encoder, nbfilters_decoder,
    batch_norm, encoder_downsampling, decoder_upsampling.
    """
    def __init__(self,
                 in_dim: Tuple[int],
                 out_dim: Tuple[int],
                 latent_dim: int = 2,
                 **kwargs) -> None:
        super(ImSpecTrainer, self).__init__()
        from ..nets import init_imspec_model
        seed = kwargs.get("seed", 1)
        kwargs["batch_seed"] = kwargs.get("batch_seed", seed)
        set_train_rng(seed)
        self.in_dim, self.out_dim = in_dim, out_dim
        self.latent_dim = latent_dim
        self.net, self.meta_state_dict = init_imspec_model(in_dim, out_dim, latent_dim, **kwargs)
        self.net.to(self.device)
        self.meta_state_dict["weights"] = self.net.state_dict()

    def set_data(self, X_train, y_train, X_test=None, y_test=None,
                 **kwargs: Union[float, int]) -> None:
        """Sets training and test data (atomai/trainers/trainer.py:800-857)."""
        if X_test is None or y_test is None:
            from sklearn.model_selection import train_test_split
            X_train, X_test, y_train, y_test = train_test_split(
                X_train, y_train, test_size=kwargs.get("test_size", .15),
                shuffle=True, random_state=kwargs.get("seed", 1))
        if self.full_epoch:
            self.train_loader, self.test_loader, dims = init_imspec_dataloaders(
                X_train, y_train, X_test, y_test, self.batch_size,
                memory_alloc=kwargs.get("memory_alloc", 4))
        else:
            (self.X_train, self.y_train, self.X_test, self.y_test,
             dims) = preprocess_training_imspec_data(
                 X_train, y_train, X_test, y_test, self.batch_size, kwargs.get("memory_alloc", 4))
        self.data_is_set = True
        if dims[0] != tuple(self.in_dim) or dims[1] != tuple(self.out_dim):
            raise AssertionError(
                "The input/output dimensions of the model must match" +
                " the height, width and length (for spectra) of training")


def _split_if_no_test(X_train, y_train, X_test, y_test, kwargs):
    if X_test is None or y_test is None:
        from sklearn.model_selection import train_test_split
        X_train, X_test, y_train, y_test = train_test_split(
            X_train, y_train, test_size=kwargs.get("test_size", .15),
            shuffle=True, random_state=kwargs.get("seed", 1))
    return X_train, y_train, X_test, y_test


class RegTrainer(BaseTrainer):
    """
    Trainer for image -> vector regression (atomai/trainers/trainer.py:860-950): out_dim, backbone
    ('mobilenet'; 'resnet' / 'vgg' raise NotImplementedError) and the kwargs input_channels,
    seed, batch_seed.  Criterion: mean squared error.
    """
    def __init__(self, out_dim: int = 1, backbone: str = "mobilenet", **kwargs) -> None:
        super(RegTrainer, self).__init__()
        from ..nets import init_reg_model
        seed = kwargs.get("seed", 1)
        kwargs["batch_seed"] = kwargs.get("batch_seed", seed)
        set_train_rng(seed)
        self.output_size = out_dim
        self.criterion = self.get_loss_fn('mse')
        self.net, self.meta_state_dict = init_reg_model(out_dim, backbone, **kwargs)
        self.net.to(self.device)
        self.meta_state_dict["weights"] = self.net.state_dict()

    def set_data(self, X_train, y_train, X_test=None, y_test=None,
                 **kwargs: Union[float, int]) -> None:
        """Images (n, c, h, w) or (n, h, w), targets (n, out_dim) or (n,); a train / test split
        (test_size, seed) when no test set is given; memory_alloc."""
        from ..utils.preproc import preprocess_training_reg_data, preprocess_training_reg_data_
        X_train, y_train, X_test, y_test = _split_if_no_test(X_train, y_train, X_test, y_test,
                                                             kwargs)
        memory_alloc = kwargs.get("memory_alloc", 4)
        if self.full_epoch:
            self.train_loader, self.test_loader = init_dataloaders(
                *preprocess_training_reg_data_(X_train, y_train, X_test, y_test),
                self.batch_size, memory_alloc)
            train_out_dim = self.train_loader.dataset.tensors[1].shape[-1]
            test_out_dim = self.test_loader.dataset.tensors[1].shape[-1]
        else:
            (self.X_train, self.y_train, self.X_test, self.y_test) = preprocess_training_reg_data(
                X_train, y_train, X_test, y_test, self.batch_size, memory_alloc)
            train_out_dim, test_out_dim = self.y_train[0].shape[-1], self.y_test[0].shape[-1]
        self.data_is_set = True
        if not train_out_dim == test_out_dim == self.output_size:
            raise AssertionError(
                "The output dimensions for the training and test data must be" +
                " equal to the declared output dimensions")


class clsTrainer(BaseTrainer):
    """
    Trainer for image classification (atomai/trainers/trainer.py:953-1046): nb_classes, backbone
    ('mobilenet'; 'resnet' / 'vgg' raise NotImplementedError) and the kwargs input_channels,
    seed, batch_seed.  Criterion: mean NLL of the network's log-probabilities (losses.NLLLoss).
    """
    def __init__(self, nb_classes: int, backbone: str = "mobilenet", **kwargs) -> None:
        super(clsTrainer, self).__init__()
        from ..nets import init_cls_model
        seed = kwargs.get("seed", 1)
        kwargs["batch_seed"] = kwargs.get("batch_seed", seed)
        set_train_rng(seed)
        self.nb_classes = nb_classes
        self.criterion = losses_metrics.NLLLoss()
        self.net, self.meta_state_dict = init_cls_model(nb_classes, backbone, **kwargs)
        self.net.to(self.device)
        if self.device == 'cpu':
            warnings.warn("No GPU found. atomai_b200 cannot train without an H100 (sm_90a)",
                          UserWarning)
        self.meta_state_dict["weights"] = self.net.state_dict()

    def set_data(self, X_train, y_train, X_test=None, y_test=None,
                 **kwargs: Union[float, int]) -> None:
        """Images (n, c, h, w) or (n, h, w) and 1-D int64 class labels; a train / test split
        (test_size, seed) when no test set is given; memory_alloc."""
        from ..utils.preproc import preprocess_training_cls_data, preprocess_training_cls_data_
        X_train, y_train, X_test, y_test = _split_if_no_test(X_train, y_train, X_test, y_test,
                                                             kwargs)
        # the NLL kernel cannot raise from the device (an out-of-range label gives a NaN loss), so
        # the labels are checked once here, on the host
        for what, y in (("training", y_train), ("test", y_test)):
            lo, hi = int(y.min()), int(y.max())
            if lo < 0 or hi >= self.nb_classes:
                raise ValueError(f"{what} labels must lie in [0, {self.nb_classes - 1}] for "
                                 f"nb_classes={self.nb_classes}, got [{lo}, {hi}]")
        memory_alloc = kwargs.get("memory_alloc", 4)
        if self.full_epoch:
            self.train_loader, self.test_loader = init_dataloaders(
                *preprocess_training_cls_data_(X_train, y_train, X_test, y_test),
                self.batch_size, memory_alloc)
        else:
            (self.X_train, self.y_train, self.X_test, self.y_test) = preprocess_training_cls_data(
                X_train, y_train, X_test, y_test, self.batch_size, memory_alloc)
        self.data_is_set = True

    def accuracy_fn(self, y: torch.Tensor, y_prob: torch.Tensor, *args):
        """Ratio of correct argmax predictions (atomai/trainers/trainer.py:1039-1046)."""
        _, predicted = torch.max(y_prob.data, 1)
        total = y.size(0)
        correct = (predicted == y).sum().item()
        return correct / total
