"""High-level fault-tolerant trainer: the "one call a user makes" per step.

Two pipelines over the same model code (``models/llama.py``):

``backend="b200"`` (default) -- FT-ZeRO-1 on the NVLink data plane (``parallel/zero1.py``)::

    ProcessGroupB200 (peer-memory kernels, remap-on-quorum)
      -> Manager (quorum / heal on the C++ control plane; commit verdict ON THE DEVICE)
      -> FlatParams: weights + gradients in flat SYMMETRIC bf16 buffers
      -> backward: per-block reduce-scatter kernel (1/N scale, zero contribution, buddy push) on the comm stream
      -> commit:   one verdict kernel (AND over the quorum through the signal pads), no host sync, no RPC
      -> update:   gated AdamW on the held slices fused with the all-gather of the new weights, block by
                   block on the optimizer stream while the next forward already runs

``backend="nccl"`` -- the reference-equivalent arm: stock ``ProcessGroupNCCL`` re-created per quorum,
per-bucket all-reduce SUM then ``/N``, host-synchronous ``should_commit`` RPC, full AdamW on every
replica (upstream torchft/manager.py:466-478,884-903, upstream torchft/optim.py:52-55).
``backend="b200"`` with ``zero1=False`` runs that same classic structure on the native all-reduce kernels.

This is the HSDP configuration of BASELINE.json with shard degree 1: every GPU is one replica group holding
the full bf16 model and its training state (on an 80 GB H100: up to ~3 B parameters), and the replicated dimension is both the fault-tolerance dimension
(README.md:37-42 of the reference) and -- new here -- the dimension the optimizer is partitioned over.
"""

from __future__ import annotations

import contextlib
import dataclasses
import os
from datetime import timedelta
from typing import Any, Callable, Dict, Iterator, List, Optional, Tuple

import torch
from torch import nn
from torch.distributed import TCPStore

from torchft_b200.data import check_cu_seqlens, slice_cu_seqlens
from torchft_b200.ddp import FlatDistributedDataParallel
from torchft_b200.manager import Manager
from torchft_b200.models.llama import CONFIGS, FlatParams, Llama, LlamaConfig
from torchft_b200.optim import OptimizerWrapper
from torchft_b200.ops.fused import FlatAdamW
from torchft_b200.parallel.zero1 import intersect_ranges, merge_ranges


def no_decay_ranges(flat: FlatParams, module: nn.Module, select: Callable[[str, nn.Parameter], bool]
                    ) -> List[Tuple[int, int]]:
    """The flat element ranges of ``module``'s parameters for which ``select(name, p)`` holds, each with the
    ``FlatParams.ALIGN`` padding behind it (the padding is never read, so exempting it changes nothing), merged."""
    where = {id(p): o for p, o in zip(flat.params, flat.offsets)}
    out = []
    for name, p in module.named_parameters():
        if id(p) in where and select(name, p):
            o = where[id(p)]
            out.append((o, min(o + (p.numel() + FlatParams.ALIGN - 1) // FlatParams.ALIGN * FlatParams.ALIGN, flat.numel)))
    return merge_ranges(out)


def fp8_linears_from_env(default: bool = False) -> bool:
    """``TORCHFT_B200_FP8``: ``"1"`` turns the fp8 block linears on, ``"0"`` turns them off, unset gives ``default``
    (the model config's setting, off unless the config asks for it); any other value raises."""
    v = os.environ.get("TORCHFT_B200_FP8")
    if v is None:
        return default
    if v not in ("0", "1"):
        raise ValueError(f"TORCHFT_B200_FP8 must be 0 or 1, got {v!r}")
    return v == "1"


class FaultTolerantTrainer:
    """Llama trainer over one replica group per GPU.

    Args:
        model: config name in ``models.llama.CONFIGS`` or a ``LlamaConfig``
        lighthouse_addr: address of a running Lighthouse
        replica_id: this replica group's name (``"replica_3"``); trailing digits give its global rank
        min_replica_size: minimum participating replicas for a step to commit
        backend: ``"b200"`` (native peer-memory kernels) or ``"nccl"`` (reference-equivalent baseline)
        zero1: partition the optimizer over the replicas and commit on the device (default for ``b200``;
            env ``TORCHFT_B200_ZERO1=0`` turns it off)
        replication: holders per slice of optimizer state (``k`` of FT-ZeRO-1)
        compact_state: FT-ZeRO-1: store only the held slices of the optimizer state, in page pools sized for every
            quorum of ``min_replica_size`` to 8 replicas (``None``: env ``TORCHFT_B200_Z1_COMPACT=1`` turns it on)
        max_grad_norm: FT-ZeRO-1: clip the global L2 norm of the reduced gradient to this, on the device; a step with a
            non-finite norm is skipped on every replica (``inf``: only that). ``None``: env
            ``TORCHFT_B200_Z1_MAX_GRAD_NORM``, unset = no clipping. Not available on the classic all-reduce pipeline.
        grad_accum_steps: FT-ZeRO-1: micro-batches per optimizer step (``M``). ``step`` and friends then take
            ``(M * B, S)`` inputs, run ``M`` forward/backward passes of ``B`` sequences and apply the gradient of the mean
            loss over all of them; each micro-batch is reduce-scattered under its own backward into an fp32
            accumulator of this replica's slices. Not available on the classic all-reduce pipeline.
        lr_lambda: FT-ZeRO-1: learning-rate schedule as a ``LambdaLR`` lambda stepped once per committed step: committed
            update ``t`` uses ``lr * lr_lambda(min(t, lr_steps) - 1)``; vetoed steps do not advance it. Tabulated once
            at construction. Not available on the classic all-reduce pipeline.
        lr_steps: FT-ZeRO-1: length of that table (required with ``lr_lambda``); later updates keep its last rate
        no_decay: FT-ZeRO-1: ``(name, parameter) -> bool`` selecting the parameters that get no weight decay, e.g.
            ``lambda name, p: p.ndim == 1`` for the norm gains. Not available on the classic all-reduce pipeline.
        moment_dtype: FT-ZeRO-1: ``torch.bfloat16`` keeps the AdamW moments in bf16 (8 instead of 12 bytes of optimizer
            state per parameter), rounded stochastically so that the holders of a slice stay bit-identical; ``None``:
            env ``TORCHFT_B200_Z1_MOMENTS=bf16``, unset = fp32. Not available on the classic all-reduce pipeline.
        ema_decay: FT-ZeRO-1: keep an exponential moving average of the fp32 master weights with this decay, as
            partitioned optimizer state of the moments' type, advanced by every committed update (``None``: env
            ``TORCHFT_B200_Z1_EMA_DECAY``, unset = no EMA). :meth:`ema_weights` evaluates it. Not available on the
            classic all-reduce pipeline.
        audit_every: FT-ZeRO-1: every ``N``-th update since the last quorum change, check on the device that every
            replica holds the same bf16 weights and the holders of each slice the same optimizer state; a disagreement
            fails the next step on every replica, and the next quorum repairs it (``Zero1Optimizer``). ``None``: env
            ``TORCHFT_B200_Z1_AUDIT_EVERY``, unset = 0, off. Not available on the classic all-reduce pipeline.
        global_token_mean: FT-ZeRO-1: apply the gradient of the mean loss over every target that is not -100, in every
            micro-batch, on every participating replica of the quorum (a healing replica contributes none), instead of
            the mean of each replica's and each micro-batch's own mean. Each micro-batch's loss is then divided by its
            ``B * S`` positions, and the commit kernel, which already exchanges the verdict, sums every replica's target
            count and loss and scales the update by ``P * M * B * S / N`` (exactly 1 when no target is ignored). ``step``
            and friends return ``sum of losses / N`` over the quorum, the same on every replica of a committed step; a
            vetoed step returns this replica's own token mean. Replicas fed batches of different shapes veto the step.
            Not available on the classic all-reduce pipeline.
        fp8_linears: run the forward and input-gradient GEMMs of the four block linears on fp8 tensor cores with
            row-scaled e4m3 operands (``LlamaConfig.fp8_linears``); weight gradients, the LM head and attention stay
            bf16, so the gradient buffer and the optimizer see bf16 exactly as without it. A model property: it applies
            to every pipeline. ``None``: env ``TORCHFT_B200_FP8`` (``1`` on, ``0`` off, anything else raises; unset: the
            config's ``fp8_linears``, off by default)
        bucket_mb: gradient bucket size for the classic (all-reduce) pipeline
        should_quantize: fused fp8 gradient all-reduce (classic pipeline)
        overlap_optimizer: classic pipeline: run AdamW stage by stage on a side stream under the next forward (default);
            ``False``: one launch after ``should_commit``
        optimizer_blocks: CTA cap of the AdamW launches (0: the kernel's default, 16 CTAs per SM); FT-ZeRO-1: of the
            update launches
    """

    def __init__(self, model: str | LlamaConfig, lighthouse_addr: str, replica_id: str = "replica_0",
                 min_replica_size: int = 1, backend: str = "b200", bucket_mb: float = 512.0,
                 should_quantize: bool = False, lr: float = 3e-4, seed: int = 0,
                 timeout: timedelta = timedelta(seconds=60), device: Optional[torch.device] = None,
                 activation_checkpoint: Optional[str] = None, init_sync: bool = False,
                 use_async_quorum: bool = True, overlap_optimizer: bool = True,
                 optimizer_blocks: int = 0, zero1: Optional[bool] = None, replication: int = 2,
                 compact_state: Optional[bool] = None, max_grad_norm: Optional[float] = None,
                 grad_accum_steps: int = 1, lr_lambda: Optional[Callable[[int], float]] = None,
                 lr_steps: Optional[int] = None,
                 no_decay: Optional[Callable[[str, nn.Parameter], bool]] = None,
                 moment_dtype: Optional[torch.dtype] = None, ema_decay: Optional[float] = None,
                 fp8_linears: Optional[bool] = None, audit_every: Optional[int] = None,
                 global_token_mean: bool = False) -> None:
        cfg = CONFIGS[model] if isinstance(model, str) else model
        if activation_checkpoint is not None:
            cfg = dataclasses.replace(cfg, activation_checkpoint=activation_checkpoint)
        if fp8_linears is None:
            fp8_linears = fp8_linears_from_env(cfg.fp8_linears)
        if bool(fp8_linears) != cfg.fp8_linears:
            cfg = dataclasses.replace(cfg, fp8_linears=bool(fp8_linears))
        self.cfg = cfg
        self.backend = backend
        if zero1 is None:
            zero1 = backend == "b200" and os.environ.get("TORCHFT_B200_ZERO1", "1") != "0" and not should_quantize
        if zero1 and backend != "b200":
            raise ValueError("zero1 needs the b200 backend")
        self.zero1 = bool(zero1)
        if max_grad_norm is not None and not self.zero1:
            raise ValueError("max_grad_norm needs the FT-ZeRO-1 pipeline (backend='b200', zero1=True)")
        if int(grad_accum_steps) != grad_accum_steps or grad_accum_steps < 1:
            raise ValueError(f"grad_accum_steps must be an integer >= 1, got {grad_accum_steps}")
        if grad_accum_steps > 1 and not self.zero1:
            raise ValueError("grad_accum_steps > 1 needs the FT-ZeRO-1 pipeline (backend='b200', zero1=True)")
        self.grad_accum_steps = int(grad_accum_steps)
        if (lr_lambda is not None or no_decay is not None) and not self.zero1:
            raise ValueError("lr_lambda and no_decay need the FT-ZeRO-1 pipeline (backend='b200', zero1=True)")
        if moment_dtype is not None and not self.zero1:
            raise ValueError("moment_dtype needs the FT-ZeRO-1 pipeline (backend='b200', zero1=True)")
        if ema_decay is not None and not self.zero1:
            raise ValueError("ema_decay needs the FT-ZeRO-1 pipeline (backend='b200', zero1=True)")
        if audit_every is not None and audit_every and not self.zero1:
            raise ValueError("audit_every needs the FT-ZeRO-1 pipeline (backend='b200', zero1=True)")
        if global_token_mean and not self.zero1:
            raise ValueError("global_token_mean needs the FT-ZeRO-1 pipeline (backend='b200', zero1=True)")
        self.global_token_mean = bool(global_token_mean)
        self._in_ema = False  # inside ema_weights(): the model holds the EMA weights
        if lr_lambda is not None and lr_steps is None:
            raise ValueError("lr_lambda needs lr_steps, the length of the schedule")
        self._micro = 0  # FT-ZeRO-1: index of the micro-batch whose backward is running
        self._steps_run = 0  # steps started by this trainer (a checkpoint restore must come first)

        # the options are checked above, before anything touches the device
        self.device = device if device is not None else torch.device("cuda", torch.cuda.current_device())
        torch.cuda.set_device(self.device)

        # the replica group's own store (group world size 1 => this process hosts it)
        self._store = TCPStore("127.0.0.1", 0, is_master=True, wait_for_workers=False)

        if backend == "b200":
            from torchft_b200.parallel.process_group_b200 import ProcessGroupB200

            self.pg: Any = ProcessGroupB200(timeout=timeout, device=self.device)
        elif backend == "nccl":
            from torchft_b200.process_group import ProcessGroupNCCL

            self.pg = ProcessGroupNCCL(timeout=timeout)
        else:
            raise ValueError(f"unknown backend {backend}")

        # build on meta, materialise directly into the flat buffers, then initialise in place
        self.model = Llama(cfg, device="meta")
        numel = sum((p.numel() + FlatParams.ALIGN - 1) // FlatParams.ALIGN * FlatParams.ALIGN for p in self.model.parameters())
        self.zopt: Any = None
        if self.zero1:
            from torchft_b200.parallel.zero1 import Zero1Optimizer

            # the optimizer owns the five symmetric flat buffers; FlatParams adopts two of them. Units (= gradient
            # buckets = update launches) are the forward stages, known once the parameters have offsets.
            self.zopt = Zero1Optimizer(self.pg, numel, lr=lr, replication=replication, blocks=optimizer_blocks or None,
                                       compact=compact_state, min_world=min_replica_size, max_grad_norm=max_grad_norm,
                                       grad_accum_steps=self.grad_accum_steps, lr_lambda=lr_lambda,
                                       lr_steps=lr_steps or 0, moment_dtype=moment_dtype, ema_decay=ema_decay,
                                       audit_every=audit_every, global_token_mean=self.global_token_mean)
            self.flat = FlatParams(self.model, grad_alloc=lambda n: self.zopt.grad, device=self.device,
                                   param_alloc=lambda n: self.zopt.param)
        else:
            grad_alloc = (lambda n: self.pg.alloc_symmetric("grads", numel * 2).view(torch.bfloat16)) if backend == "b200" else None
            self.flat = FlatParams(self.model, grad_alloc=grad_alloc, device=self.device)
        self.model.init_weights(seed)
        self._stage_ranges = self._compute_stage_ranges()

        if self.zero1:
            nd = None
            if no_decay is not None:
                nd = [r for unit in self._stage_ranges
                      for r in intersect_ranges(no_decay_ranges(self.flat, self.model, no_decay), [unit])]
            self.zopt.set_units(self._stage_ranges, no_decay=nd)
            self.zopt.seed_master()
            self.inner_optim: Any = self.zopt
        else:
            self.inner_optim = FlatAdamW(self.flat.param, self.flat.grad, lr=lr)
            self.inner_optim.direct_grads = True  # step_device() drops p.grad; wgrad GEMMs fill the flat buffer

        self.manager = Manager(
            pg=self.pg,
            load_state_dict=self.load_state_dict,
            state_dict=self.state_dict,
            min_replica_size=min_replica_size,
            use_async_quorum=use_async_quorum,
            timeout=timeout,
            quorum_timeout=timeout,
            connect_timeout=timeout,
            rank=0,
            world_size=1,
            store_addr="127.0.0.1",
            store_port=self._store.port,
            lighthouse_addr=lighthouse_addr,
            replica_id=replica_id,
            init_sync=init_sync,
        )
        self._opt_stream: Optional[torch.cuda.Stream] = None
        self._opt_pending = False
        # tied embeddings with gradient accumulation: the event the head's forward write into the tied slot waits for
        self._head_after: Optional[torch.cuda.Event] = None
        if self.zero1:
            self.ddp = FlatDistributedDataParallel(self.manager, self.model, self.flat,
                                                   bucket_ranges=sorted(self._stage_ranges), reduce_fn=self._reduce_unit)
            self._bucket_unit = {bi: self._stage_ranges.index((lo, hi))
                                 for bi, (lo, hi) in enumerate(sorted(self._stage_ranges))}
            self._setup_stage_gates()
            self.zopt.bind_stream(self._opt_stream)
            self.optim: Any = None
        else:
            self.ddp = FlatDistributedDataParallel(self.manager, self.model, self.flat, bucket_mb=bucket_mb,
                                                   should_quantize=should_quantize)
            self.optim = OptimizerWrapper(self.manager, self.inner_optim)
            self._opt_blocks = int(optimizer_blocks)
            if overlap_optimizer:
                self._setup_stage_gates()
        self._tok: Optional[torch.Tensor] = None
        self._tgt: Optional[torch.Tensor] = None
        self._loss_host: Optional[torch.Tensor] = None
        self._loss_event: Optional[torch.cuda.Event] = None

    # ------------------------------------------------- stages: optimizer units == forward gates
    def _compute_stage_ranges(self) -> List[Tuple[int, int]]:
        """Element range of the flat buffer per top-level module, in FORWARD order; the ranges tile the buffer."""
        where = {id(p): (o, p.numel()) for p, o in zip(self.flat.params, self.flat.offsets)}
        ranges = []
        for stage in self.model.param_stages():
            mine = [where[id(p)] for p in stage]
            lo = min(o for o, _ in mine)
            hi = max((o + n + FlatParams.ALIGN - 1) // FlatParams.ALIGN * FlatParams.ALIGN for o, n in mine)
            ranges.append((lo, min(hi, self.flat.numel)))
        covered = sorted(ranges)
        assert covered[0][0] == 0 and covered[-1][1] == self.flat.numel and all(
            a[1] == b[0] for a, b in zip(covered, covered[1:])), "parameter stages must tile the flat buffer"
        return ranges

    def _setup_stage_gates(self) -> None:
        """The update of stage ``i`` runs on a side stream and records ``events[i]``; the NEXT forward of stage ``i``
        waits for exactly that event. The update is HBM/NVLink-bound and the forward tensor-core-bound, so they
        overlap instead of idling the tensor cores for the whole update."""
        self._opt_ranges = self._stage_ranges
        self._opt_events = [torch.cuda.Event() for _ in self._stage_ranges]
        self._opt_stream = torch.cuda.Stream(device=self.device)

        head_stage = len(self._stage_ranges) - 1

        def gate(stage: int) -> None:
            if self._opt_pending:
                torch.cuda.current_stream().wait_event(self._opt_events[stage])
            if stage == head_stage and self._head_after is not None:
                torch.cuda.current_stream().wait_event(self._head_after)

        self.model.stage_hook = gate

    # ------------------------------------------------- FT-ZeRO-1 pipeline pieces
    def _reduce_unit(self, bucket: int, start: int, end: int) -> Any:
        m = self.manager
        unit = self._bucket_unit[bucket]
        if self.grad_accum_steps == 1:
            return m.guarded(lambda: self.zopt.reduce_scatter(unit, 1.0 / max(m.num_participants(), 1), m.is_participating()))
        micro, steps = self._micro, self.grad_accum_steps
        return m.guarded(lambda: self.zopt.reduce_scatter(unit, 1.0 / (max(m.num_participants(), 1) * steps),
                                                          m.is_participating(), micro))

    # ------------------------------------------------- classic pipeline pieces
    def _optimizer_step(self) -> None:
        if self._opt_stream is None:
            self.inner_optim.step()
            return
        self._opt_stream.wait_stream(torch.cuda.current_stream())
        self.inner_optim.step_ranges(self._opt_ranges, (self._opt_stream, self._opt_events), max_blocks=self._opt_blocks)
        self._opt_pending = True

    def _join_optimizer(self) -> None:
        """Make the current stream (and later host readers) see a fully applied update."""
        if self._opt_stream is not None and self._opt_pending:
            torch.cuda.current_stream().wait_stream(self._opt_stream)

    def join(self) -> None:
        """Order the current stream behind everything the last step enqueued on side streams (the optimizer
        update / weight all-gather), e.g. before recording a timing event or reading the weights."""
        self._join_optimizer()

    # -------------------------------------------------------------- heal hooks
    def state_dict(self) -> Dict[str, Any]:
        if self._opt_stream is not None:
            self._opt_stream.synchronize()  # heal senders read on their own stream: hand them a finished update
        if self.zero1:
            return self.zopt.state_dict()
        o = self.inner_optim
        return {"param": self.flat.param, "master": o.master, "m": o.m, "v": o.v, "t": o.t}

    def load_state_dict(self, sd: Dict[str, Any]) -> None:
        self._join_optimizer()
        if self.zero1:
            self.zopt.load_state_dict(sd)
            return
        o = self.inner_optim
        with torch.no_grad():
            for name, dst in (("param", self.flat.param), ("master", o.master), ("m", o.m), ("v", o.v)):
                if sd[name].data_ptr() != dst.data_ptr():
                    dst.copy_(sd[name])
        o.t = int(sd["t"])

    # -------------------------------------------------------------------- step
    def step_device(self, tokens: torch.Tensor, targets: torch.Tensor,
                    cu_seqlens: Optional[torch.Tensor] = None) -> torch.Tensor:
        """One fault-tolerant optimisation step on device-resident inputs; returns the loss tensor (device). With
        ``grad_accum_steps = M`` the inputs are ``(M * B, S)`` and the loss is the mean over the ``M`` micro-batches.
        ``cu_seqlens`` (host int32, ``data.check_cu_seqlens``) packs documents into the rows (``Llama.forward``); with
        accumulation it describes the whole ``(M * B, S)`` batch and is cut per micro-batch on the host."""
        self._not_in_ema("step")
        self._steps_run += 1
        if self.zero1 and self.grad_accum_steps > 1:
            return self._step_accumulate(tokens, targets, cu_seqlens)
        if self.zero1:
            self.manager.start_quorum()       # async; its thread first books the previous step's device verdict
            self.flat.reset_grads()           # wgrad GEMMs write the flat gradient buffer directly: no memset
            loss = self.ddp(tokens, targets, cu_seqlens=cu_seqlens,  # forward; stage i waits for unit i's update
                            **self._loss_kw())
            loss.backward()                   # per-unit reduce-scatter kernels launch from the grad hooks
            self.ddp.finish(wait=False)       # issue what is left; the optimizer stream orders itself behind them
            if self.global_token_mean:
                self._publish_tokens(targets, [loss], tokens.numel())
            self.manager.commit_on_device(self.zopt)  # verdict kernel (no host sync, no RPC in steady state)
            self.zopt.update(self._opt_events)        # gated AdamW + weight all-gather, unit by unit
            self._opt_pending = True
            return self.zopt.token_mean_loss() if self.global_token_mean else loss
        self.optim.zero_grad(set_to_none=True)  # start_quorum (async); no memset:
        self.flat.reset_grads()                  # wgrad GEMMs write the flat gradient buffer directly
        loss = self.ddp(tokens, targets, cu_seqlens=cu_seqlens)  # forward (fused kernels + cuBLAS + SDPA)
        loss.backward()                   # bucket all-reduces launch from grad hooks, overlapped
        self.ddp.finish()                 # current stream waits for the comm stream
        if self.manager.should_commit():  # OptimizerWrapper.step() semantics (optim.py), with the update
            self._optimizer_step()        # cut per layer so the next forward overlaps it
        return loss

    def _step_accumulate(self, tokens: torch.Tensor, targets: torch.Tensor,
                         cu_seqlens: Optional[torch.Tensor] = None) -> torch.Tensor:
        """FT-ZeRO-1 step over ``M`` micro-batches: one quorum, ``M`` forward/backward passes whose reduce-scatters
        accumulate on the comm stream, one commit and one update.

        By default the loss (and its gradient) is the mean of the ``M`` micro-batch means, each over its own targets that
        are not -100, not the mean over all valid targets of the step, and the replicas are averaged alike. With packed
        documents the number of valid targets varies more between micro-batches (one -100 per document, and a padded
        tail), so a target in a micro-batch of many short documents weighs more than one in a micro-batch of few long
        ones. With ``global_token_mean`` each micro-batch's loss is its sum over ``B * S`` instead, and the commit kernel
        rescales the reduced gradient to the mean over every valid target of every micro-batch on every participating
        replica: ``M`` micro-batches of ``B`` rows then take the step one batch of ``M * B`` rows takes, and so do
        replicas with different masks. The loss returned is that global mean."""
        M = self.grad_accum_steps
        if tokens.shape[0] % M or tokens.shape[0] == 0 or targets.shape[0] != tokens.shape[0]:
            raise ValueError(f"grad_accum_steps={M} must divide the batch dimension of tokens and targets, got "
                             f"{tuple(tokens.shape)} and {tuple(targets.shape)}")
        B = tokens.shape[0] // M
        micro_cu: List[Optional[torch.Tensor]] = [None] * M
        if cu_seqlens is not None:
            S = tokens.shape[1]
            check_cu_seqlens(cu_seqlens, M * B, S)  # row-aligned, so every micro-batch boundary is a document start
            micro_cu = [slice_cu_seqlens(cu_seqlens, m * B * S, (m + 1) * B * S) for m in range(M)]
        cur = torch.cuda.current_stream()
        read_done = torch.cuda.Event()
        tied = self.cfg.tie_embeddings
        losses = []
        self.manager.start_quorum()              # once: the quorum is fixed for all micro-batches of the step
        for m in range(M):
            self._micro = m
            self.flat.reset_grads()
            # tied: the head writes its dW into the tied slot during the FORWARD, while the peers may still read that
            # slot for micro-batch m-1's tied unit, the last reduce-scatter of its backward. The head's stage waits for
            # the same event as the backward below; the blocks' forward still overlaps that reduce-scatter.
            self._head_after = read_done if tied and m > 0 else None
            try:
                loss = self.ddp(tokens[m * B:(m + 1) * B], targets[m * B:(m + 1) * B],  # overlaps micro-batch m-1's tail
                                cu_seqlens=micro_cu[m], **self._loss_kw())
            finally:
                self._head_after = None
            if m > 0:
                # backward overwrites the gradient buffer that the peers read in micro-batch m-1's reduce-scatters:
                # wait until its last trailing handshake ("every peer is done reading mine") has passed
                cur.wait_event(read_done)
            loss.backward()
            self.ddp.finish(wait=False)
            if m < M - 1:
                read_done.record(self.pg.comm_stream)
            losses.append(loss.detach().float())
        if self.global_token_mean:
            self._publish_tokens(targets, losses, B * tokens.shape[1])
        self.manager.commit_on_device(self.zopt)
        self.zopt.update(self._opt_events)
        self._opt_pending = True
        if self.global_token_mean:
            return self.zopt.token_mean_loss()
        return torch.stack(losses).mean()

    def _loss_kw(self) -> Dict[str, Any]:
        """Global token mean: each micro-batch's loss is its sum over its ``B * S`` positions, a divisor every replica
        shares; the commit kernel turns the reduced gradient into the mean over the quorum's valid targets."""
        return {"count_valid": False} if self.global_token_mean else {}

    def _publish_tokens(self, targets: torch.Tensor, losses: List[torch.Tensor], c: int) -> None:
        """Hand the commit this step's count of valid targets (over the whole ``(M * B, S)`` input) and its loss sum
        ``sum_m loss_m * c`` in fp64, added in micro-batch order as the commit kernel adds the replicas in rank order."""
        n = (targets != -100).sum()
        total: Optional[torch.Tensor] = None
        for loss in losses:
            x = loss.detach().double() * c
            total = x if total is None else total + x
        assert total is not None
        m = self.manager
        self.zopt.publish_tokens(n, total, targets.numel(), max(m.num_participants(), 1), m.is_participating())

    def _stage_inputs(self, tokens_cpu: torch.Tensor, targets_cpu: torch.Tensor) -> None:
        B, S = tokens_cpu.shape
        if self._tok is None or self._tok.shape != tokens_cpu.shape:
            self._tok = torch.empty((B, S), dtype=torch.int64, device=self.device)
            self._tgt = torch.empty((B, S), dtype=torch.int64, device=self.device)
        assert self._tgt is not None
        self._tok.copy_(tokens_cpu, non_blocking=True)
        self._tgt.copy_(targets_cpu, non_blocking=True)

    def step(self, tokens_cpu: torch.Tensor, targets_cpu: torch.Tensor,
             cu_seqlens: Optional[torch.Tensor] = None) -> float:
        """End-to-end step: pinned-host inputs -> H2D -> train step -> D2H loss (blocks until the loss is on the host).
        ``cu_seqlens``: packed documents, as in :meth:`step_device`."""
        self._not_in_ema("step")
        self._stage_inputs(tokens_cpu, targets_cpu)
        loss = self.step_device(self._tok, self._tgt, cu_seqlens)
        return float(loss.item())

    def step_async(self, tokens_cpu: torch.Tensor, targets_cpu: torch.Tensor,
                   cu_seqlens: Optional[torch.Tensor] = None) -> Optional[float]:
        """Like :meth:`step`, but the loss comes back one step late: this call enqueues the step and the D2H copy
        of ITS loss into pinned memory, and returns the PREVIOUS step's loss (``None`` on the first call). The host
        never waits for the step it just launched, so the GPU queue stays full; every step still performs its
        H2D input copy and its D2H loss read. ``cu_seqlens``: packed documents, as in :meth:`step_device`."""
        self._not_in_ema("step_async")
        prev: Optional[float] = None
        if self._loss_event is not None:
            self._loss_event.synchronize()
            assert self._loss_host is not None
            prev = float(self._loss_host[0])
        self._stage_inputs(tokens_cpu, targets_cpu)
        loss = self.step_device(self._tok, self._tgt, cu_seqlens)
        if self._loss_host is None:
            self._loss_host = torch.empty(1, dtype=torch.float32).pin_memory()
            self._loss_event = torch.cuda.Event()
        self._loss_host.copy_(loss.detach().float().reshape(1), non_blocking=True)
        self._loss_event.record()
        return prev

    # ----------------------------------------------------- durable checkpoints (FT-ZeRO-1)
    def _require_zero1_ckpt(self) -> None:
        if not self.zero1:
            raise ValueError("save_checkpoint / restore_checkpoint need the FT-ZeRO-1 pipeline (backend='b200', "
                             "zero1=True); the classic pipeline keeps its full optimizer state on every replica and "
                             "checkpoints with checkpointing.DurableCheckpointer")

    def save_checkpoint(self, directory: str, keep: int = 2) -> int:
        """Write this replica's share of a durable checkpoint of the last committed step to ``directory`` (shared by
        every replica of the job) and return its step ``T`` once the write is enqueued. Call it on every replica after
        the same step. The copy to host memory runs under the next step's forward and backward; the file is written by
        a background thread (:meth:`wait_checkpoint`). The ``keep`` newest steps this replica wrote are kept."""
        self._require_zero1_ckpt()
        self._not_in_ema("save_checkpoint")
        ms = self.manager.state_dict()  # settles the last step's deferred verdict: the host learns T, no other sync
        assert ms["step"] == self.zopt.t, (ms, self.zopt.t)
        return self.zopt.save(directory, ms, self._opt_events, keep)

    def wait_checkpoint(self) -> None:
        """Block until the last :meth:`save_checkpoint` is on disk; raises if the write failed."""
        self._require_zero1_ckpt()
        self.zopt.wait_checkpoint()

    def restore_checkpoint(self, directory: str) -> Optional[int]:
        """Before the first step: resume from the newest complete checkpoint in ``directory``. Returns its step, or
        ``None`` when there is none (a fresh run). Works at any number of replicas: ranges a live replica of the same
        step still holds are pulled from it at the first quorum, the rest are read from the files. The data loader's
        position is the caller's to restore from the returned step."""
        self._require_zero1_ckpt()
        if self._steps_run:
            raise RuntimeError("restore_checkpoint must be called before the first step")
        ms = self.zopt.restore(directory)
        if ms is None:
            return None
        self.manager.load_state_dict(ms)
        return int(ms["step"])

    # ----------------------------------------------------- EMA of the weights (FT-ZeRO-1)
    @contextlib.contextmanager
    def ema_weights(self) -> Iterator[None]:
        """Evaluate the EMA of the weights: inside the context ``self.model`` holds bf16(EMA) (e.g. ``with
        torch.no_grad(): trainer.model(tokens)``); on exit it holds the training weights again, bit for bit. Every
        replica enters after the same step. :meth:`step`, :meth:`step_device`, :meth:`step_async` and
        :meth:`save_checkpoint` raise inside it."""
        if self.zopt is None or self.zopt.ema is None:
            raise RuntimeError("ema_weights needs the FT-ZeRO-1 pipeline with an ema_decay")
        self._not_in_ema("ema_weights")
        self.join()  # the last step's update has finished before its EMA is read
        with self.zopt.ema_weights():
            self._in_ema = True
            try:
                yield
            finally:
                self._in_ema = False

    def _not_in_ema(self, what: str) -> None:
        if self._in_ema:
            raise RuntimeError(f"{what} inside ema_weights(): the model holds the EMA weights, not the training weights")

    def last_grad_norm(self) -> Optional[float]:
        """Global gradient norm of the most recently resolved step (FT-ZeRO-1 with clipping; ``None`` otherwise). Steps
        resolve lazily, so after step ``n`` this is usually the norm of step ``n - 1``."""
        return self.zopt.last_grad_norm if self.zopt is not None else None

    def last_lr(self) -> Optional[float]:
        """The fp32 learning rate of the most recently resolved committed update (FT-ZeRO-1; ``None`` before the first
        one and on the classic pipeline). Steps resolve lazily, like :meth:`last_grad_norm`."""
        if self.zopt is None or self.zopt.t < 1:
            return None
        return self.zopt.lr_at(self.zopt.t)

    def last_loss(self) -> Optional[float]:
        """Loss of the most recent :meth:`step_async` (waits for it)."""
        if self._loss_event is None:
            return None
        self._loss_event.synchronize()
        assert self._loss_host is not None
        return float(self._loss_host[0])

    def shutdown(self) -> None:
        if self._opt_stream is not None:
            self._opt_stream.synchronize()
        if self.zopt is not None:
            self.zopt.wait_checkpoint()  # a checkpoint write in flight lands (or raises) before the process moves on
        self.manager.shutdown(wait=False)
        self.pg.shutdown()
