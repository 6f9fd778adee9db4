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

import dataclasses
import os
from datetime import timedelta
from typing import Any, Dict, List, Optional, Tuple

import torch
from torch.distributed import TCPStore

from torchft_b200.ddp import FlatDistributedDataParallel
from torchft_b200.manager import Manager
from torchft_b200.models.llama import CONFIGS, FlatParams, Llama, LlamaConfig
from torchft_b200.optim import OptimizerWrapper
from torchft_b200.ops.fused import FlatAdamW


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
        bucket_mb: gradient bucket size for the classic (all-reduce) pipeline
        should_quantize: fused fp8 gradient all-reduce (classic pipeline)
        overlap_optimizer: classic pipeline: run AdamW stage by stage on a side stream under the next forward
    """

    def __init__(self, model: str | LlamaConfig, lighthouse_addr: str, replica_id: str = "replica_0",
                 min_replica_size: int = 1, backend: str = "b200", bucket_mb: float = 512.0,
                 should_quantize: bool = False, lr: float = 3e-4, seed: int = 0,
                 timeout: timedelta = timedelta(seconds=60), device: Optional[torch.device] = None,
                 activation_checkpoint: Optional[str] = None, init_sync: bool = False,
                 use_async_quorum: bool = True, overlap_optimizer: Optional[bool] = None,
                 optimizer_blocks: int = 0, zero1: Optional[bool] = None, replication: int = 2) -> None:
        self.device = device if device is not None else torch.device("cuda", torch.cuda.current_device())
        torch.cuda.set_device(self.device)
        cfg = CONFIGS[model] if isinstance(model, str) else model
        if activation_checkpoint is not None:
            cfg = dataclasses.replace(cfg, activation_checkpoint=activation_checkpoint)
        self.cfg = cfg
        self.backend = backend
        if zero1 is None:
            zero1 = backend == "b200" and os.environ.get("TORCHFT_B200_ZERO1", "1") != "0" and not should_quantize
        if zero1 and backend != "b200":
            raise ValueError("zero1 needs the b200 backend")
        self.zero1 = bool(zero1)

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
            self.zopt = Zero1Optimizer(self.pg, numel, lr=lr, replication=replication, blocks=optimizer_blocks or None)
            self.flat = FlatParams(self.model, grad_alloc=lambda n: self.zopt.grad, device=self.device,
                                   param_alloc=lambda n: self.zopt.param)
        else:
            grad_alloc = (lambda n: self.pg.alloc_symmetric("grads", numel * 2).view(torch.bfloat16)) if backend == "b200" else None
            self.flat = FlatParams(self.model, grad_alloc=grad_alloc, device=self.device)
        self.model.init_weights(seed)
        self._stage_ranges = self._compute_stage_ranges()

        if self.zero1:
            self.zopt.set_units(self._stage_ranges)
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
            if overlap_optimizer is None:
                overlap_optimizer = os.environ.get("TORCHFT_B200_OVERLAP_OPT", "1") != "0"
            self._opt_blocks = int(os.environ.get("TORCHFT_B200_OPT_BLOCKS", optimizer_blocks))
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

        def gate(stage: int) -> None:
            if self._opt_pending:
                torch.cuda.current_stream().wait_event(self._opt_events[stage])

        self.model.stage_hook = gate

    # ------------------------------------------------- FT-ZeRO-1 pipeline pieces
    def _reduce_unit(self, bucket: int, start: int, end: int) -> Any:
        m = self.manager
        unit = self._bucket_unit[bucket]
        return m.guarded(lambda: self.zopt.reduce_scatter(unit, 1.0 / max(m.num_participants(), 1), m.is_participating()))

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
    def step_device(self, tokens: torch.Tensor, targets: torch.Tensor) -> torch.Tensor:
        """One fault-tolerant optimisation step on device-resident inputs; returns the loss tensor (device)."""
        if self.zero1:
            self.manager.start_quorum()       # async; its thread first books the previous step's device verdict
            self.flat.reset_grads()           # wgrad GEMMs write the flat gradient buffer directly: no memset
            loss = self.ddp(tokens, targets)  # forward; stage i waits for the event of unit i's update
            loss.backward()                   # per-unit reduce-scatter kernels launch from the grad hooks
            self.ddp.finish(wait=False)       # issue what is left; the optimizer stream orders itself behind them
            self.manager.commit_on_device(self.zopt)  # verdict kernel (no host sync, no RPC in steady state)
            self.zopt.update(self._opt_events)        # gated AdamW + weight all-gather, unit by unit
            self._opt_pending = True
            return loss
        self.optim.zero_grad(set_to_none=True)  # start_quorum (async); no memset:
        self.flat.reset_grads()                  # wgrad GEMMs write the flat gradient buffer directly
        loss = self.ddp(tokens, targets)  # forward (fused kernels + cuBLAS + SDPA)
        loss.backward()                   # bucket all-reduces launch from grad hooks, overlapped
        self.ddp.finish()                 # current stream waits for the comm stream
        if self.manager.should_commit():  # OptimizerWrapper.step() semantics (optim.py), with the update
            self._optimizer_step()        # cut per layer so the next forward overlaps it
        return loss

    def _stage_inputs(self, tokens_cpu: torch.Tensor, targets_cpu: torch.Tensor) -> None:
        B, S = tokens_cpu.shape
        if self._tok is None or self._tok.shape != tokens_cpu.shape:
            self._tok = torch.empty((B, S), dtype=torch.int64, device=self.device)
            self._tgt = torch.empty((B, S), dtype=torch.int64, device=self.device)
        assert self._tgt is not None
        self._tok.copy_(tokens_cpu, non_blocking=True)
        self._tgt.copy_(targets_cpu, non_blocking=True)

    def step(self, tokens_cpu: torch.Tensor, targets_cpu: torch.Tensor) -> float:
        """End-to-end step: pinned-host inputs -> H2D -> train step -> D2H loss (blocks until the loss is on the host)."""
        self._stage_inputs(tokens_cpu, targets_cpu)
        loss = self.step_device(self._tok, self._tgt)
        return float(loss.item())

    def step_async(self, tokens_cpu: torch.Tensor, targets_cpu: torch.Tensor) -> Optional[float]:
        """Like :meth:`step`, but the loss comes back one step late: this call enqueues the step and the D2H copy
        of ITS loss into pinned memory, and returns the PREVIOUS step's loss (``None`` on the first call). The host
        never waits for the step it just launched, so the GPU queue stays full; every step still performs its
        H2D input copy and its D2H loss read."""
        prev: Optional[float] = None
        if self._loss_event is not None:
            self._loss_event.synchronize()
            assert self._loss_host is not None
            prev = float(self._loss_host[0])
        self._stage_inputs(tokens_cpu, targets_cpu)
        loss = self.step_device(self._tok, self._tgt)
        if self._loss_host is None:
            self._loss_host = torch.empty(1, dtype=torch.float32).pin_memory()
            self._loss_event = torch.cuda.Event()
        self._loss_host.copy_(loss.detach().float().reshape(1), non_blocking=True)
        self._loss_event.record()
        return prev

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
        self.manager.shutdown(wait=False)
        self.pg.shutdown()
