"""
viBaseTrainer — training loop of the variational autoencoders with the reference's interface
(atomai/trainers/vitrainer.py:19-396): set_model / set_data / compile_trainer / reparameterize /
train_epoch / evaluate_model / save_model.  Encoder, decoder, reconstruction loss and the Adam step
run as native sm_90a kernels; under torchrun the DataLoader batches are sharded over the ranks and
the gradients all-reduced once per step (the encoder's fc weights dominate: ~21 MB per step).
"""
from typing import Callable, Optional, Tuple, Type, Union

import numpy as np
import torch

from ..optim import FusedAdam
from ..parallel import Comm, GradBucket, broadcast_model
from ..utils.nn import reset_bnorm, set_train_rng, weights_init
from ..utils.preproc import get_array_memsize


class viBaseTrainer:
    """Initializes base trainer for VAE and VED models."""
    def __init__(self):
        set_train_rng(1)
        self.device = "cuda" if torch.cuda.is_available() else "cpu"
        self.in_dim = None
        self.out_dim = None
        self.z_dim = 1
        self.encoder_net = None
        self.decoder_net = None
        self.train_iterator = None
        self.test_iterator = None
        self.aux_model_params = []
        self.optim = None
        self.current_epoch = 0
        self.metadict = {}
        self.loss_history = {"train_loss": [], "test_loss": []}
        self.filename = "model"
        self.training_cycles = 1
        self.batch_size = 1
        self.comm: Optional[Comm] = None
        self._bucket: Optional[GradBucket] = None

    def set_model(self, encoder_net: Type[torch.nn.Module],
                  decoder_net: Type[torch.nn.Module]) -> None:
        self.encoder_net = encoder_net.to(self.device)
        self.decoder_net = decoder_net.to(self.device)

    def set_encoder(self, encoder_net: Type[torch.nn.Module]) -> None:
        self.encoder_net = encoder_net.to(self.device)

    def set_decoder(self, decoder_net: Type[torch.nn.Module]) -> None:
        self.decoder_net = decoder_net.to(self.device)

    def set_data(self, X_train, y_train=None, X_test=None, y_test=None,
                 memory_alloc: float = 4) -> None:
        """Initializes train and (optionally) test data loaders (vitrainer.py:83-99)."""
        arrsize = sum(get_array_memsize(x) for x in (X_train, y_train, X_test, y_test))
        store_on_cpu = (arrsize / 1e9) > memory_alloc
        self.train_iterator = self._set_data(X_train, y_train, store_on_cpu)
        if X_test is not None:
            self.test_iterator = self._set_data(X_test, y_test, store_on_cpu)

    def _2torch(self, X, y=None) -> Tuple[torch.Tensor]:
        if isinstance(X, np.ndarray):
            X = torch.from_numpy(X)
        if isinstance(y, np.ndarray):
            y = torch.from_numpy(y)
        return X, y

    def _set_data(self, X, y=None, store_on_cpu: bool = False):
        """TensorDataset + DataLoader(shuffle=True, drop_last=True) (vitrainer.py:101-124)."""
        if X is None:
            raise AssertionError("You must provide input train/test data")
        device_ = 'cpu' if store_on_cpu else self.device
        X, y = self._2torch(X, y)
        X = X.to(device_)
        y = y.to(device_) if y is not None else y
        data = torch.utils.data.TensorDataset(X, y) if y is not None \
            else torch.utils.data.TensorDataset(X,)
        return torch.utils.data.DataLoader(data, batch_size=self.batch_size, shuffle=True,
                                           drop_last=True)

    def elbo_fn(self):
        raise NotImplementedError

    def forward_compute_elbo(self):
        raise NotImplementedError

    def _reset_rng(self, seed: int) -> None:
        set_train_rng(seed)

    def _reset_weights(self) -> None:
        for net in (self.encoder_net, self.decoder_net):
            net.apply(weights_init)
            net.apply(reset_bnorm)

    def _reset_training_history(self) -> None:
        self.loss_history = {"train_loss": [], "test_loss": []}

    def _delete_optimizer(self) -> None:
        self.optim = None

    def compile_trainer(self, train_data, test_data=None,
                        optimizer: Optional[Type[torch.optim.Optimizer]] = None,
                        elbo_fn: Callable = None, training_cycles: int = 100,
                        batch_size: int = 32, **kwargs: Union[str, float]) -> None:
        """Compiles model's trainer (vitrainer.py:173-221); default optimizer Adam(lr=1e-4),
        here the fused multi-tensor kernel.  kwargs: filename, memory_alloc."""
        self.training_cycles = training_cycles
        self.batch_size = batch_size
        if elbo_fn is not None:
            self.elbo_fn = elbo_fn
        alloc = kwargs.get("memory_alloc", 4)
        if torch.distributed.is_available() and torch.distributed.is_initialized() \
                and torch.distributed.get_world_size() > 1:
            self.comm = Comm()
            if batch_size % self.comm.world != 0:
                raise ValueError("batch_size must be divisible by the number of ranks")
        if test_data is not None:
            self.set_data(*train_data, *test_data, memory_alloc=alloc)
        else:
            self.set_data(*train_data, memory_alloc=alloc)
        params = list(self.decoder_net.parameters()) + list(self.encoder_net.parameters())
        for aux_param in self.aux_model_params:
            params.extend(list(aux_param))
        if self.comm is not None:
            broadcast_model(self.encoder_net, self.comm)
            broadcast_model(self.decoder_net, self.comm)
        if self.optim is None:
            if optimizer is None:
                self.optim = FusedAdam(params, lr=1e-4) if self.device == "cuda" \
                    else torch.optim.Adam(params, lr=1e-4)
            else:
                self.optim = optimizer(params)
        if self.comm is not None:
            self._bucket = GradBucket(params)
            if isinstance(self.optim, FusedAdam):
                self.optim.grad_scale = 1.0 / self.comm.world
                self._bucket.post_scale = 1.0
            else:
                self._bucket.post_scale = 1.0 / self.comm.world
        self.filename = kwargs.get("filename", "./model")

    @classmethod
    def reparameterize(cls, z_mean: torch.Tensor, z_sd: torch.Tensor) -> torch.Tensor:
        """z = mu + sd * eps, eps ~ N(0, 1) (vitrainer.py:223-234); (B, latent)-sized torch op."""
        return z_mean + z_sd * torch.randn_like(z_mean)

    def _shard(self, x):
        if self.comm is None or self.comm.world == 1:
            return x
        k = x.shape[0] // self.comm.world
        return x[self.comm.rank * k:(self.comm.rank + 1) * k]

    def train_epoch(self):
        """Trains a single epoch; returns the running mean of the ELBO (vitrainer.py:292-318)."""
        if self.device != "cuda":
            raise RuntimeError("atomai_b200 trains on CUDA (sm_90a) only; there is no CPU path")
        step = self.forward_compute_elbo
        self.decoder_net.train()
        self.encoder_net.train()
        c, elbo_epoch = 0, 0
        for x in self.train_iterator:
            if len(x) == 1:
                x, y = self._shard(x[0].to(self.device)), None
            else:
                x, y = self._shard(x[0].to(self.device)), self._shard(x[1].to(self.device))
            b = x.size(0)
            if self._bucket is not None:
                self._bucket.zero_()
            elbo = step(x) if y is None else step(x, y)
            loss = -elbo
            loss.backward()
            if self._bucket is not None:
                self._bucket.attach()
                self._bucket.allreduce(self.comm)
            self.optim.step()
            self.optim.zero_grad(set_to_none=self._bucket is None)
            elbo = elbo.item()
            c += b
            elbo_epoch += b * (elbo - elbo_epoch) / c
        return elbo_epoch

    def evaluate_model(self):
        """Evaluates model on test data (vitrainer.py:320-345)."""
        step = self.forward_compute_elbo
        self.decoder_net.eval()
        self.encoder_net.eval()
        c, elbo_epoch_test = 0, 0
        for x in self.test_iterator:
            if len(x) == 1:
                x, y = x[0].to(self.device), None
            else:
                x, y = x[0].to(self.device), x[1].to(self.device)
            b = x.size(0)
            elbo = step(x, mode="eval") if y is None else step(x, y, mode="eval")
            elbo = elbo.item()
            c += b
            elbo_epoch_test += b * (elbo - elbo_epoch_test) / c
        return elbo_epoch_test

    def print_statistics(self, e):
        if self.comm is not None and self.comm.rank != 0:
            return
        if self.test_iterator is not None:
            print('Epoch: {}/{}, Training loss: {:.4f}, Test loss: {:.4f}'.format(
                e + 1, self.training_cycles, -self.loss_history["train_loss"][-1],
                -self.loss_history["test_loss"][-1]))
        else:
            print('Epoch: {}/{}, Training loss: {:.4f}'.format(
                e + 1, self.training_cycles, -self.loss_history["train_loss"][-1]))

    def save_model(self, *args: str) -> None:
        """Saves encoder/decoder weights, optimizer and the meta-dict as `<name>.tar`
        (vitrainer.py:361-372)."""
        savepath = args[0] if len(args) > 0 else self.filename
        self.metadict["encoder"] = self.encoder_net.state_dict()
        self.metadict["decoder"] = self.decoder_net.state_dict()
        self.metadict["optimizer"] = self.optim
        if self.comm is None or self.comm.rank == 0:
            torch.save(self.metadict, savepath + ".tar")

    def save_weights(self, *args: str) -> None:
        savepath = args[0] if len(args) > 0 else self.filename + "weights"
        torch.save({"encoder": self.encoder_net.state_dict(),
                    "decoder": self.decoder_net.state_dict()}, savepath + ".tar")

    def load_weights(self, filepath: str) -> None:
        weights = torch.load(filepath, map_location=self.device)
        self.encoder_net.load_state_dict(weights["encoder"])
        self.decoder_net.load_state_dict(weights["decoder"])
