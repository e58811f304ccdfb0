"""Input pipeline helpers for 3-D parallel jobs on GPUs.

The reference leaves data loading to the user's script: a ``DistributedSampler(num_replicas=dp_size,
rank=ctx.get_local_rank(ParallelMode.DATA))`` and a blocking ``.to("cuda")`` per step (reference
examples/hybrid_parallelism.py:39-63, tests/convergence/run_hybrid_parallel.py).  Getting the sampler's two numbers
wrong is the classic 3-D-parallel bug — ranks of one tensor / pipeline group must read the SAME batch, replicas
different ones — so this module owns them:

* :func:`data_parallel_sampler` / :func:`build_dataloader` — sharded over the DATA group only, seeded identically on
  every rank, pinned host memory when the job runs on GPUs;
* :class:`TokenFileDataset` — fixed-length sequences over a flat binary token file (``numpy.memmap``: the page cache is
  the only copy on the host, nothing is tokenised or collated per step);
* :class:`DevicePrefetcher` — keeps ``depth`` batches in flight to the device on a copy stream (pinned host buffer →
  ``cudaMemcpyAsync`` → event), so the H2D transfer of step ``i + 1`` overlaps the kernels of step ``i`` and the
  compute stream only ever waits on an event.  A 64 KB batch of token ids is latency-, not bandwidth-bound
  (≈ 10 µs), which is exactly why it must not sit on the compute stream between two steps.
"""
from __future__ import annotations

from collections import deque
from typing import Dict, Iterable, Iterator, Optional, Union

import torch
from torch.utils.data import DataLoader, Dataset, DistributedSampler

from pipegoose_b200.constants import SEED
from pipegoose_b200.distributed.parallel_mode import ParallelMode


def data_parallel_sampler(dataset, parallel_context, shuffle: bool = True, seed: int = SEED,
                          drop_last: bool = False) -> DistributedSampler:
    """The sampler of a 3-D parallel job: one shard per data-parallel replica — every rank of a replica's tensor and
    pipeline groups gets the same indices in the same order (``seed`` must be the same on all ranks; it is by default)."""
    return DistributedSampler(dataset, num_replicas=parallel_context.get_world_size(ParallelMode.DATA),
                              rank=parallel_context.get_local_rank(ParallelMode.DATA), shuffle=shuffle, seed=seed,
                              drop_last=drop_last)


def build_dataloader(dataset, parallel_context, batch_size: int, shuffle: bool = True, seed: int = SEED,
                     drop_last: bool = True, num_workers: int = 0, collate_fn=None, prefetch_to_device: bool = True,
                     prefetch_depth: int = 2):
    """``DataLoader`` over this replica's shard; on a GPU job the batches are collated into pinned memory and (with
    ``prefetch_to_device``) arrive on the rank's device through a :class:`DevicePrefetcher`.  ``loader.sampler`` is the
    :func:`data_parallel_sampler` (the ``Trainer`` calls its ``set_epoch``)."""
    sampler = data_parallel_sampler(dataset, parallel_context, shuffle=shuffle, seed=seed, drop_last=drop_last)
    device = getattr(parallel_context, "device", None)
    on_gpu = isinstance(device, torch.device) and device.type == "cuda" and torch.cuda.is_available()
    loader = DataLoader(dataset, batch_size=batch_size, sampler=sampler, drop_last=drop_last, num_workers=num_workers,
                        collate_fn=collate_fn, pin_memory=on_gpu, persistent_workers=num_workers > 0)
    if on_gpu and prefetch_to_device:
        return DevicePrefetcher(loader, device, depth=prefetch_depth)
    return loader


class TokenFileDataset(Dataset):
    """Sequences of ``seq_len`` tokens over a flat file of token ids (``uint16`` / ``uint32`` / ``int64``, the layout
    ``write_token_file`` and most pre-tokenised corpora use).  Item ``i`` is tokens ``[i * stride, i * stride + seq_len)``
    as ``{"input_ids": int64[seq_len]}`` (the models shift the labels themselves: pass ``labels=input_ids``).

    ``eos_token_id``: the file is a concatenation of documents, each ended by this token.  Every item then also carries
    ``"position_ids"`` (int64 ``[seq_len]``): 0 at the window's first token, +1 per token, back to 0 on the token after
    each ``eos_token_id`` (the eos belongs to the document it ends).  The models then keep the documents of a window
    from attending to each other and from predicting each other's tokens; a ``Trainer`` passes the item to the model
    as it is."""

    def __init__(self, path: str, seq_len: int, dtype: str = "uint16", stride: Optional[int] = None,
                 eos_token_id: Optional[int] = None):
        import numpy as np

        self.path, self.seq_len = path, int(seq_len)
        self.eos_token_id = None if eos_token_id is None else int(eos_token_id)
        self.stride = int(stride) if stride is not None else self.seq_len
        self.dtype = np.dtype(dtype)
        self._tokens = None            # opened lazily: a memmap must not be pickled into DataLoader workers
        n = np.memmap(path, dtype=self.dtype, mode="r").shape[0]
        if n < self.seq_len:
            raise ValueError(f"{path} holds {n} tokens, fewer than one sequence of {self.seq_len}")
        self.n_tokens = int(n)
        self._len = (n - self.seq_len) // self.stride + 1

    def __len__(self) -> int:
        return self._len

    def _open(self):
        import numpy as np

        if self._tokens is None:
            self._tokens = np.memmap(self.path, dtype=self.dtype, mode="r")
        return self._tokens

    def __getitem__(self, i: int) -> Dict[str, torch.Tensor]:
        import numpy as np

        if i < 0:
            i += self._len
        if not 0 <= i < self._len:
            raise IndexError(i)
        start = i * self.stride
        chunk = np.asarray(self._open()[start:start + self.seq_len]).astype(np.int64)
        item = {"input_ids": torch.from_numpy(chunk)}
        if self.eos_token_id is not None:
            item["position_ids"] = torch.from_numpy(_packed_positions(chunk, self.eos_token_id))
        return item

    def __getstate__(self):
        state = dict(self.__dict__)
        state["_tokens"] = None
        return state


def _packed_positions(tokens, eos_token_id: int):
    """int64 positions of a window of concatenated documents: ``arange`` restarted after every ``eos_token_id``."""
    import numpy as np

    n = tokens.shape[0]
    idx = np.arange(n, dtype=np.int64)
    start = np.zeros(n, dtype=np.int64)
    start[1:] = np.where(tokens[:-1] == eos_token_id, idx[1:], 0)
    return idx - np.maximum.accumulate(start)


def write_token_file(path: str, tokens: Union[torch.Tensor, Iterable[int]], dtype: str = "uint16") -> None:
    """Flat binary token file for :class:`TokenFileDataset` (ids must fit ``dtype``)."""
    import numpy as np

    arr = tokens.detach().cpu().numpy() if isinstance(tokens, torch.Tensor) else np.asarray(list(tokens))
    info = np.iinfo(np.dtype(dtype))
    if arr.size and (arr.min() < info.min or arr.max() > info.max):
        raise ValueError(f"token ids {arr.min()}..{arr.max()} do not fit {dtype}")
    arr.astype(dtype).tofile(path)


def _to_device(obj, device, pin: bool):
    if isinstance(obj, torch.Tensor):
        if pin and obj.device.type == "cpu" and not obj.is_pinned():
            obj = obj.pin_memory()
        return obj.to(device, non_blocking=True)
    if isinstance(obj, dict):
        return {k: _to_device(v, device, pin) for k, v in obj.items()}
    if isinstance(obj, (list, tuple)):
        return type(obj)(_to_device(v, device, pin) for v in obj)
    return obj


def _record_stream(obj, stream):
    if isinstance(obj, torch.Tensor):
        if obj.is_cuda:
            obj.record_stream(stream)
    elif isinstance(obj, dict):
        for v in obj.values():
            _record_stream(v, stream)
    elif isinstance(obj, (list, tuple)):
        for v in obj:
            _record_stream(v, stream)


class DevicePrefetcher:
    """Iterate ``loader`` with ``depth`` batches already on their way to ``device``.

    GPU: copies are issued on a private stream from pinned memory; ``__next__`` makes the caller's current stream wait on
    the batch's event (no host synchronisation) and marks the tensors as used by that stream so the caching allocator
    does not recycle them under the step.  CPU (tests, gloo dry runs): the same look-ahead without streams.
    ``bytes_per_batch`` reports what one batch moved (the ``h2d_bytes_per_step`` of ``bench.py``'s end-to-end number)."""

    def __init__(self, loader: Iterable, device: Union[str, torch.device], depth: int = 2):
        assert depth >= 1
        self.loader = loader
        self.device = torch.device(device)
        self.depth = depth
        self._cuda = self.device.type == "cuda" and torch.cuda.is_available()
        self._stream = torch.cuda.Stream(device=self.device) if self._cuda else None
        self.bytes_per_batch = 0

    # what a Trainer looks at on its loader
    @property
    def sampler(self):
        return getattr(self.loader, "sampler", None)

    @property
    def dataset(self):
        return getattr(self.loader, "dataset", None)

    def __len__(self) -> int:
        return len(self.loader)

    def _stage(self, batch):
        self.bytes_per_batch = _nbytes(batch)
        if not self._cuda:
            return _to_device(batch, self.device, pin=False), None
        with torch.cuda.stream(self._stream):
            moved = _to_device(batch, self.device, pin=True)
            event = torch.cuda.Event()
            event.record(self._stream)
        return moved, event

    def __iter__(self) -> Iterator:
        source = iter(self.loader)
        queue: deque = deque()

        def fill():
            while len(queue) < self.depth:
                try:
                    queue.append(self._stage(next(source)))
                except StopIteration:
                    return

        fill()
        while queue:
            batch, event = queue.popleft()
            if event is not None:
                current = torch.cuda.current_stream(self.device)
                current.wait_event(event)
                _record_stream(batch, current)
            fill()          # the next copy is in flight before the caller starts computing on this batch
            yield batch


def _nbytes(obj) -> int:
    if isinstance(obj, torch.Tensor):
        return obj.numel() * obj.element_size()
    if isinstance(obj, dict):
        return sum(_nbytes(v) for v in obj.values())
    if isinstance(obj, (list, tuple)):
        return sum(_nbytes(v) for v in obj)
    return 0
