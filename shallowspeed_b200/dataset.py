"""Dataset: MNIST-shaped data, DP-sharded and micro-batched.

Parity with the reference's ``Dataset`` (``shallowspeed/dataset.py:5-86``): constructor
``Dataset(save_dir, global_batch_size, mubatch_size, validation)``, ``load(DP_rank,
DP_size)`` truncates to a multiple of the global batch and takes the rank-strided slice
``[DP_rank::DP_size]`` (so global batch b is samples ``[b*GBS, (b+1)*GBS)`` of the file
on ANY layout -> DP == sequential), ``load_micro_batch_input/target(batch_id,
mubatch_id)`` return contiguous row slices, ``get_num_batches``, ``get_num_mubatches``,
``len``.

GPU-first additions: the GPU machines may have no network, so the dataset can
be *synthetic* (``synthetic_mnist``: class-conditional prototypes + noise with MNIST's
shape, split sizes and normalisation - learnable, so accuracy curves still mean
something); the shard lives either in pinned host memory (end-to-end path: one H2D copy
per step) or resident in HBM (``device=...``; 59 500 x 784 fp32 = 187 MB, nothing next to
80 GB); ``write_reference_files`` stores any dataset in the reference's on-disk format
(x_{split}.parquet + y_{split}.npy) so the unmodified reference can train on identical
data.

Shuffling (``shuffle_seed=...``, training data only): every rank keeps the whole file, and
global position q of epoch e (``set_epoch``) holds row ``shuffle_index(N, seed, e, q)`` of
it (``ops.functional``: a keyed Feistel permutation of [0, N)).  Local row n of DP rank r
in global batch b stays position ``b * GBS + n * dp + r``; an epoch has ``N // GBS``
batches, and the ``N mod GBS`` positions past the last one are dropped (different samples
every epoch).  ``shuffle_seed=None`` is the unshuffled layout above.
"""
from __future__ import annotations

from pathlib import Path
from typing import Optional

import numpy as np
import torch

from .ops import functional as F

N_TRAIN, N_VAL, N_FEATURES, N_CLASSES = 59500, 10500, 784, 10  # reference download_dataset.py:16-18


def synthetic_mnist(validation: bool = False, n: Optional[int] = None, n_features: int = N_FEATURES,
                    n_classes: int = N_CLASSES, seed: int = 42):
    """Deterministic MNIST-shaped data: x = clip(prototype[class] + noise) / 255 - mean."""
    n = n if n is not None else (N_VAL if validation else N_TRAIN)
    rs = np.random.RandomState(seed)
    protos = rs.uniform(0.0, 255.0, (n_classes, n_features)).astype(np.float32)
    protos *= (rs.uniform(0, 1, (n_classes, n_features)) < 0.25)          # sparse strokes like digits
    rs2 = np.random.RandomState(seed + (1 if validation else 2))
    labels = rs2.randint(0, n_classes, n)
    x = protos[labels] + rs2.normal(0.0, 64.0, (n, n_features)).astype(np.float32)
    x = np.clip(x, 0.0, 255.0) / np.float32(255.0)
    x -= np.float32(0.1307)                                                # MNIST global mean
    y = np.zeros((n, n_classes), dtype=np.float32)
    y[np.arange(n), labels] = 1.0
    return x.astype(np.float32), y


def write_reference_files(save_dir, overwrite: bool = False, **kw):
    """Write synthetic data in the reference's file format (dataset.py:43-47)."""
    import pandas as pd

    save_dir = Path(save_dir)
    save_dir.mkdir(parents=True, exist_ok=True)
    for split, val in (("train", False), ("val", True)):
        xp, yp = save_dir / f"x_{split}.parquet", save_dir / f"y_{split}.npy"
        if xp.exists() and yp.exists() and not overwrite:
            continue
        x, y = synthetic_mnist(validation=val, **kw)
        pd.DataFrame(x, columns=[f"pixel{i}" for i in range(x.shape[1])]).to_parquet(xp)
        np.save(yp, y)
    return save_dir


class Dataset:
    def __init__(self, save_dir, global_batch_size, mubatch_size, validation=False,
                 synthetic: Optional[bool] = None, device=None, pin_memory: bool = False,
                 n_samples: Optional[int] = None, n_features: int = N_FEATURES, n_classes: int = N_CLASSES,
                 shuffle_seed: Optional[int] = None):
        self.shuffle_seed = F.check_shuffle_seed(shuffle_seed)
        if validation and self.shuffle_seed is not None:
            raise ValueError("a validation dataset is never shuffled (shuffle_seed must be None)")
        self.epoch = 0
        self.dp_rank, self.dp_size = 0, 1
        self._ids = None          # (epoch, batch_id, file rows of the local batch on the data's device)
        if save_dir is not None:
            save_dir = Path(save_dir)
        if synthetic is None:
            synthetic = save_dir is None or not (save_dir / ("x_val.parquet" if validation else "x_train.parquet")).exists()
        if not synthetic:
            assert save_dir.is_dir(), "Download the dataset first! (or pass synthetic=True)"
        self.save_dir = save_dir
        self.synthetic = synthetic
        self.global_batch_size = global_batch_size
        self.local_batch_size = None
        self.mubatch_size = mubatch_size
        self._val = validation
        self.device = torch.device(device) if device is not None else torch.device("cpu")
        self.pin_memory = pin_memory
        self._n, self._nf, self._nc = n_samples, n_features, n_classes
        self.input_X: Optional[torch.Tensor] = None
        self.target_y: Optional[torch.Tensor] = None

    # -- loading ------------------------------------------------------------
    def _read_all(self):
        if self.synthetic:
            return synthetic_mnist(self._val, n=self._n, n_features=self._nf, n_classes=self._nc)
        import pandas as pd

        suffix = "val" if self._val else "train"
        x = pd.read_parquet(self.save_dir / f"x_{suffix}.parquet").to_numpy(dtype=np.float32)
        y = np.load(self.save_dir / f"y_{suffix}.npy").astype(np.float32)
        return x, y

    def load(self, DP_rank, DP_size):
        assert DP_rank < DP_size
        assert self.global_batch_size % DP_size == 0
        assert (self.global_batch_size // DP_size) % self.mubatch_size == 0, "μBatchsize must divide batchsize!"
        self.local_batch_size = self.global_batch_size // DP_size
        self.dp_rank, self.dp_size = int(DP_rank), int(DP_size)
        x, y = self._read_all()
        assert len(x) == len(y)
        if self.shuffle:   # every rank keeps the whole file: the permutation picks any row for any rank
            return self.from_arrays(x, y, DP_rank=DP_rank, DP_size=DP_size)
        full = len(x) - (len(x) % self.global_batch_size)
        return self.from_arrays(x[DP_rank:full:DP_size], y[DP_rank:full:DP_size])

    def from_arrays(self, x, y, DP_rank=None, DP_size=None):
        """Install an already sharded (x, y) pair (numpy or torch).  A shuffled dataset installs the whole file instead,
        and ``DP_rank`` / ``DP_size`` name the rank whose rows it serves (default: the ones recorded before)."""
        if DP_size is not None:
            assert 0 <= DP_rank < DP_size and self.global_batch_size % DP_size == 0
            self.dp_rank, self.dp_size = int(DP_rank), int(DP_size)
            self.local_batch_size = self.global_batch_size // DP_size
        if self.local_batch_size is None:
            self.local_batch_size = self.global_batch_size
        xt = torch.as_tensor(np.ascontiguousarray(x) if isinstance(x, np.ndarray) else x, dtype=torch.float32).contiguous()
        yt = torch.as_tensor(np.ascontiguousarray(y) if isinstance(y, np.ndarray) else y, dtype=torch.float32).contiguous()
        if self.device.type != "cpu":
            xt, yt = xt.to(self.device), yt.to(self.device)
        elif self.pin_memory and torch.cuda.is_available():
            xt, yt = xt.pin_memory(), yt.pin_memory()
        self.input_X, self.target_y = xt, yt
        self._ids = None
        if self.shuffle:
            assert self.local_batch_size % self.mubatch_size == 0
            assert len(xt) == len(yt) and self.global_batch_size <= len(xt) < 2 ** 32, "need 1 <= N // GBS and N < 2**32"
            return self
        assert len(self.input_X) % self.mubatch_size == 0
        assert len(self.input_X) % self.local_batch_size == 0
        return self

    # -- shuffling ----------------------------------------------------------
    @property
    def shuffle(self) -> bool:
        return self.shuffle_seed is not None

    def set_epoch(self, epoch: int):
        """The epoch whose permutation the batches follow from now on (used mod 2**32), like
        ``DistributedSampler.set_epoch``.  No effect on an unshuffled dataset."""
        if isinstance(epoch, bool) or not isinstance(epoch, int) or epoch < 0:
            raise ValueError(f"epoch must be an integer >= 0, got {epoch!r}")
        self.epoch = int(epoch)

    def sample_ids(self, batch_id, mubatch_id=None) -> torch.Tensor:
        """Rows of the file (int64, on the data's device) that this rank's local batch ``batch_id`` holds - or its micro-batch
        ``mubatch_id``: local row n is global position q = batch_id * GBS + n * dp + rank, the file row
        ``shuffle_index(N, seed, epoch, q)`` when shuffled and q itself otherwise."""
        assert 0 <= batch_id < self.get_num_batches()
        key = (self.epoch, batch_id)
        if self._ids is None or self._ids[0] != key:
            q = batch_id * self.global_batch_size + torch.arange(self.local_batch_size) * self.dp_size + self.dp_rank
            ids = F.shuffle_index(len(self.input_X), self.shuffle_seed, self.epoch, q) if self.shuffle else q
            self._ids = (key, ids.to(self.input_X.device))
        ids = self._ids[1]
        if mubatch_id is None:
            return ids
        assert 0 <= mubatch_id < self.get_num_mubatches()
        return ids[mubatch_id * self.mubatch_size:(mubatch_id + 1) * self.mubatch_size]

    # -- access -------------------------------------------------------------
    def __len__(self):
        return len(self.input_X)

    def _range(self, batch_id, mubatch_id):
        assert batch_id < self.get_num_batches()
        assert mubatch_id < self.get_num_mubatches()
        start = batch_id * self.local_batch_size + mubatch_id * self.mubatch_size
        end = start + self.mubatch_size
        assert end <= len(self.input_X)
        return start, end

    def load_micro_batch_input(self, batch_id, mubatch_id):
        if self.shuffle:
            return self.input_X.index_select(0, self.sample_ids(batch_id, mubatch_id))
        s, e = self._range(batch_id, mubatch_id)
        return self.input_X[s:e]

    def load_micro_batch_target(self, batch_id, mubatch_id):
        if self.shuffle:
            return self.target_y.index_select(0, self.sample_ids(batch_id, mubatch_id))
        s, e = self._range(batch_id, mubatch_id)
        return self.target_y[s:e]

    def load_batch(self, batch_id):
        """The whole DP-local batch (all micro-batches) - what the native engine stages
        with one copy per step (a shuffled dataset: gathered rows, which the native engine
        gathers itself on the device instead)."""
        if self.shuffle:
            ids = self.sample_ids(batch_id)
            return self.input_X.index_select(0, ids), self.target_y.index_select(0, ids)
        s = batch_id * self.local_batch_size
        return self.input_X[s : s + self.local_batch_size], self.target_y[s : s + self.local_batch_size]

    def get_num_batches(self):
        if self.shuffle:
            return len(self) // self.global_batch_size
        return len(self) // self.local_batch_size

    def get_num_mubatches(self):
        return self.local_batch_size // self.mubatch_size
