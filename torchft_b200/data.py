"""Data sharding across replica groups (reference: upstream torchft/data.py:24-77), and packed documents.

Fault tolerance keeps the WORLD elastic, so the dataset is sharded over the
*maximum* grid ``num_replica_groups x num_replicas``; when a replica group is down
its shard is simply skipped for those steps. For exactly-once semantics pair this
with a stateful dataloader checkpointed next to ``Manager.state_dict()``.
"""

from __future__ import annotations

from typing import Iterable, Iterator, List, Optional, Sequence, Tuple

import numpy as np
import torch
import torch.distributed as dist
from torch.utils import data


class DistributedSampler(data.distributed.DistributedSampler):
    """Sampler for worker ``group_rank`` of replica group ``replica_rank``.

    global rank  = group_rank + num_replicas * replica_rank
    global world = num_replicas * num_replica_groups
    """

    def __init__(self, dataset: data.Dataset, replica_rank: int, num_replica_groups: int,
                 group_rank: Optional[int] = None, num_replicas: Optional[int] = None, **kwargs: object) -> None:
        if group_rank is None:
            group_rank = dist.get_rank()
        if num_replicas is None:
            num_replicas = dist.get_world_size()
        self.global_rank: int = group_rank + num_replicas * replica_rank
        self.global_world_size: int = num_replicas * num_replica_groups
        super().__init__(dataset, rank=self.global_rank, num_replicas=self.global_world_size, **kwargs)  # type: ignore[arg-type]


# ------------------------------------------------------------------------------------------------- packed documents
# A batch of packed documents is ``tokens [B, S]`` plus ``cu_seqlens``: a CPU int32 tensor ``[N + 1]`` of document starts
# over the flattened ``B * S`` tokens, ``0 = c_0 < c_1 < ... < c_N = B * S``, that contains every row start ``k * S`` (no
# document crosses a row, so a micro-batch of whole rows is described by a slice of it). It stays on the host: the loader
# makes it there, and the longest document, which the attention kernel needs as a Python int, is then known without a
# device sync.


def check_cu_seqlens(cu_seqlens: object, batch: int, seq_len: int) -> int:
    """Raise ``ValueError`` naming the broken rule unless ``cu_seqlens`` describes documents of a ``(batch, seq_len)``
    token batch as above; return the length of the longest document."""
    if not isinstance(cu_seqlens, torch.Tensor):
        raise ValueError(f"cu_seqlens must be a torch.Tensor, got {type(cu_seqlens).__name__}")
    if cu_seqlens.dtype != torch.int32:
        raise ValueError(f"cu_seqlens must be int32, got {cu_seqlens.dtype}")
    if cu_seqlens.device.type != "cpu":
        raise ValueError(f"cu_seqlens must be a CPU tensor (host metadata), got device {cu_seqlens.device}")
    if cu_seqlens.dim() != 1 or cu_seqlens.numel() < 2:
        raise ValueError(f"cu_seqlens must be 1-D with at least 2 entries, got shape {tuple(cu_seqlens.shape)}")
    total = batch * seq_len
    c = cu_seqlens.numpy().astype(np.int64)
    if c[0] != 0:
        raise ValueError(f"cu_seqlens must start at 0, got {int(c[0])}")
    if c[-1] != total:
        raise ValueError(f"cu_seqlens must end at B*S = {total}, got {int(c[-1])}")
    lengths = np.diff(c)
    if (lengths <= 0).any():
        i = int(np.argmax(lengths <= 0))
        raise ValueError(f"cu_seqlens must be strictly increasing, got {int(c[i])} then {int(c[i + 1])} at index {i}")
    missing = np.setdiff1d(np.arange(0, total, seq_len), c)
    if missing.size:
        raise ValueError(f"cu_seqlens must contain every row start k*S (S = {seq_len}), so that no document crosses a "
                         f"row; missing {missing[:4].tolist()}")
    return int(lengths.max())


def document_positions(cu_seqlens: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """int32 ``[c_N]``: each token's offset in its document, ``t - c_i`` for ``c_i <= t < c_{i+1}`` (the RoPE
    position). ``out``, when given, receives it (e.g. a slice of a pinned staging buffer)."""
    c = cu_seqlens.numpy().astype(np.int64)
    starts = np.repeat(c[:-1], np.diff(c))
    pos = np.arange(c[-1], dtype=np.int64) - starts
    if out is None:
        out = torch.empty(int(c[-1]), dtype=torch.int32)
    out.numpy()[:] = pos
    return out


def slice_cu_seqlens(cu_seqlens: torch.Tensor, start: int, end: int) -> torch.Tensor:
    """The description of tokens ``[start, end)`` of a valid ``cu_seqlens`` whose documents do not cross ``start`` or
    ``end`` (row boundaries always qualify), re-based so that it starts at 0."""
    keep = (cu_seqlens >= start) & (cu_seqlens <= end)
    return (cu_seqlens[keep] - start).to(torch.int32)


def pack_documents(documents: Iterable[Sequence[int]], batch: int, seq_len: int
                   ) -> Iterator[Tuple[torch.Tensor, torch.Tensor, torch.Tensor]]:
    """Pack 1-D token sequences, in order, into batches of ``batch`` rows of ``seq_len`` tokens; yields ``(tokens
    [batch, seq_len] int64, targets [batch, seq_len] int64, cu_seqlens int32)``, all on the CPU (pin them yourself).

    Rules:

    * Documents are laid down back to back, row by row; every row start begins a document.
    * Within a document each target is the next token of the same document; the last token of a document has target
      ``-100``, so no token is trained to predict the next document.
    * A document longer than what is left of the current row is split there: the first piece fills the row and the
      rest continues at the start of the next row (or the next batch) as a new document, so its positions restart at 0.
      The last token of a piece that is continued keeps its real target, the first token of the continuation.
    * When the documents run out, the rest of the last batch is one padding document per row (token 0, every target
      ``-100``). A batch is only yielded if it holds at least one real token.
    * Empty documents are skipped. The output depends only on the inputs.
    """
    if batch < 1 or seq_len < 1:
        raise ValueError(f"batch and seq_len must be >= 1, got {batch} and {seq_len}")
    total = batch * seq_len
    tok = np.zeros(total, dtype=np.int64)
    tgt = np.full(total, -100, dtype=np.int64)
    starts: List[int] = []
    fill = 0

    def flush() -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        nonlocal tok, tgt, starts, fill
        # padding: the unfilled tail of the current row is one document, every later row another
        cut = sorted(set(starts) | set(range(0, total, seq_len)) | ({fill} if fill < total else set()))
        out = (torch.from_numpy(tok.reshape(batch, seq_len)), torch.from_numpy(tgt.reshape(batch, seq_len)),
               torch.tensor(cut + [total], dtype=torch.int32))
        tok = np.zeros(total, dtype=np.int64)
        tgt = np.full(total, -100, dtype=np.int64)
        starts, fill = [], 0
        return out

    for doc in documents:
        d = np.asarray(doc, dtype=np.int64).reshape(-1)
        i = 0
        while i < d.size:
            room = seq_len - fill % seq_len
            n = min(room, d.size - i)
            starts.append(fill)
            tok[fill:fill + n] = d[i:i + n]
            tgt[fill:fill + n] = d[i + 1:i + n + 1] if i + n < d.size else np.append(d[i + 1:i + n], -100)
            fill += n
            i += n
            if fill == total:
                yield flush()
    if fill:
        yield flush()
