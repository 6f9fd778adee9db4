"""Communication-efficient fault-tolerant algorithms: LocalSGD and (Streaming) DiLoCo.

Semantics follow upstream torchft/local_sgd.py (context managers driven by
inner-optimizer step hooks; quorum at the start of every sync window; on any
failure the window is discarded and parameters reset to the last global copy;
DiLoCo needs a synchronous quorum; fragments sync round-robin, prepared
``fragment_sync_delay`` steps before they are applied; ``fragment_update_alpha``
mixes local and global weights; the backup copy and the outer optimizer travel
with live heals).

What is different (native):

* every fragment keeps its pseudo-gradients in ONE flat buffer; parameters see
  views of it, so "bucketization" is a slicing decision, not a pack/unpack copy
  (reference packs into a fresh buffer and unpacks in a future callback,
  local_sgd.py:498-555);
* on ``ProcessGroupB200`` the pseudo-gradient ``original - local``, the fp8
  quantisation, the all-to-all/all-gather and the dequantisation run as ONE kernel
  over NVLink peer memory (``Manager.allreduce_delta``) -- the reference does the
  subtraction eagerly, then 3 Triton kernels + 2 NCCL collectives per call;
* LocalSGD averages parameters in place in the flat send buffer (no per-parameter clone).
"""

from __future__ import annotations

import logging
import math
import os
import time
from contextlib import nullcontext
from types import TracebackType
from typing import Any, Dict, List, Optional, Tuple, Type

import torch
from torch import nn, optim
from torch.distributed import Work
from torch.utils.hooks import RemovableHandle

from torchft_b200.manager import Manager
from torchft_b200.work import DummyWork

try:
    from torch.distributed.tensor import DTensor
except Exception:  # pragma: no cover
    DTensor = None  # type: ignore[assignment,misc]

logger = logging.getLogger(__name__)
_TRACE = os.environ.get("TORCHFT_B200_DILOCO_TRACE", "0") == "1"  # print the duration of every phase of an outer sync


def _trace(tag: str, t0: float) -> float:
    """With TORCHFT_B200_DILOCO_TRACE=1: drain the device, print the time since ``t0``, return the new origin."""
    if not _TRACE:
        return t0
    if torch.cuda.is_available():
        torch.cuda.synchronize()
    t1 = time.perf_counter()
    print(f"[diloco trace] {tag}: {(t1 - t0) * 1e3:.2f} ms", flush=True)
    return t1


USE_BUCKETIZATION_ENV = "TORCHFT_USE_BUCKETIZATION"


def _is_dtensor(t: Any) -> bool:
    return DTensor is not None and isinstance(t, DTensor)


def extract_local_tensor(t: torch.Tensor) -> torch.Tensor:
    """Detached clone of ``t`` (of its local shard when ``t`` is a DTensor)."""

    src = t.to_local() if _is_dtensor(t) else t
    out = src.detach().clone()
    out.grad = None
    return out


def _local_view(t: torch.Tensor) -> torch.Tensor:
    return t.to_local() if _is_dtensor(t) else t


def _assign(p: torch.Tensor, local_value: torch.Tensor, non_blocking: bool = False) -> None:
    """``p.data <- local_value`` where ``local_value`` is the local shard for DTensor params."""
    _local_view(p.data).copy_(local_value, non_blocking=non_blocking)


class LocalSGD:
    """Periodic fault-tolerant parameter averaging (https://arxiv.org/abs/1805.09767).

        with LocalSGD(manager, model, optimizer, sync_every=32):
            for batch in data:
                optimizer.zero_grad(); loss(model(batch)).backward(); optimizer.step()

    Every ``sync_every`` inner steps: quorum, all-reduce(AVG) of the parameters,
    ``should_commit``; on commit the averaged weights are written back, otherwise
    the window's progress is kept locally and the next window retries.
    """

    def __init__(self, manager: Manager, model: nn.Module, optimizer: optim.Optimizer, sync_every: int) -> None:
        assert sync_every >= 1, "sync_every must be greater than or equal to 1"
        self._manager = manager
        self._model = model
        self._local_optimizer = optimizer
        self._sync_every = sync_every
        self._local_step = 0
        self._hooks: List[RemovableHandle] = []

    def __enter__(self) -> "LocalSGD":
        self._hooks.append(self._local_optimizer.register_step_pre_hook(self._step_pre_hook))
        self._hooks.append(self._local_optimizer.register_step_post_hook(self._step_post_hook))
        return self

    def __exit__(self, exc_type: Optional[Type[BaseException]], exc_value: Optional[BaseException],
                 traceback: Optional[TracebackType]) -> bool:
        for h in self._hooks:
            h.remove()
        self._hooks.clear()
        return False

    def _step_pre_hook(self, _optim: optim.Optimizer, _args: Tuple[Any, ...], _kwargs: Dict[str, Any]) -> None:
        # a healing peer may be reading our state_dict: fence it out while weights change
        self._manager.disallow_state_dict_read()

    def _step_post_hook(self, _optim: optim.Optimizer, _args: Tuple[Any, ...], _kwargs: Dict[str, Any]) -> None:
        self._manager.allow_state_dict_read()
        self._local_step += 1
        if self._local_step >= self._sync_every:
            self.sync()

    def sync(self) -> None:
        """Average the model weights across the current quorum."""
        self._manager.start_quorum()
        self._perform_sync()
        self._local_step = 0

    def _perform_sync(self) -> None:
        averaged = self._average()
        if self._manager.should_commit():
            with torch.no_grad():
                for p, avg in zip(self._model.parameters(), averaged):
                    _assign(p, avg)

    def _average(self) -> List[torch.Tensor]:
        """All-reduce(AVG) a flat copy of the parameters; returns per-parameter views of the result."""
        params = [_local_view(p.data) for p in self._model.parameters()]
        works: List[Work] = []
        out: List[torch.Tensor] = []
        # group by (dtype, device) so each group is one flat message
        groups: Dict[Tuple[torch.dtype, torch.device], List[int]] = {}
        for i, p in enumerate(params):
            groups.setdefault((p.dtype, p.device), []).append(i)
        views: Dict[int, torch.Tensor] = {}
        for (dt, dev), idxs in groups.items():
            sizes = [(params[i].numel() + 7) // 8 * 8 for i in idxs]
            flat = torch.empty(sum(sizes), dtype=dt, device=dev)
            off = 0
            for i, sz in zip(idxs, sizes):
                v = flat[off : off + params[i].numel()].view(params[i].shape)
                v.copy_(params[i])
                views[i] = v
                off += sz
            works.append(self._manager.allreduce(flat))
        for w in works:
            w.wait()
        for i in range(len(params)):
            out.append(views[i])
        return out


class _StreamingDiLoCoFragment:
    bucket_cap_mb: int = 1 * 1024 * 1024 * 1024  # bytes, name kept for reference parity
    use_bucketization: bool = False

    def __init__(self, manager: Manager, model_fragment: nn.Module, fragment_id: int, fragment_sync_offset: int,
                 inner_optimizer: optim.Optimizer, outer_optimizer: optim.Optimizer, sync_every: int,
                 backup_device: Optional[torch.device] = None, pin_memory: bool = True,
                 use_bucketization: bool = False, bucket_cap_mb: Optional[int] = None, should_quantize: bool = False,
                 fragment_sync_delay: int = 0, fragment_update_alpha: float = 0.0) -> None:
        if fragment_sync_offset > sync_every:
            raise ValueError("Fragment must be synced once before `sync_every` steps")
        assert sync_every >= 1, "sync_every must be greater than or equal to 1"
        self._fragment_id = fragment_id
        self._manager = manager
        self._model_fragment = model_fragment
        self._fragment_sync_offset = fragment_sync_offset
        self._local_optimizer = inner_optimizer
        self._outer_optimizer = outer_optimizer
        self._sync_every = sync_every
        self._backup_device = backup_device
        self._pin_memory = pin_memory
        self._fragment_sync_delay = fragment_sync_delay
        self._fragment_update_alpha = fragment_update_alpha
        self.should_quantize = should_quantize
        if bucket_cap_mb is not None:
            self.bucket_cap_mb = int(bucket_cap_mb * 1024 * 1024)
        self.use_bucketization = os.getenv(USE_BUCKETIZATION_ENV, "False") == "True" or use_bucketization

        self._allreduce_work: List[Work] = []
        self._stream: Optional[torch.cuda.Stream] = torch.cuda.Stream() if torch.cuda.is_available() else None
        self._stop_event: Optional[torch.cuda.Event] = None
        # recorded by prepare_sync behind the pseudo-gradient all-reduce, and with it every read of the live weights; the
        # next inner optimizer step waits for it before it writes the weights
        self._read_event: Optional[torch.cuda.Event] = None

        self._names: List[str] = []
        self._params: List[torch.Tensor] = []
        # last committed global weights (restored when a sync fails), on backup_device
        self.original_parameters: Dict[str, torch.Tensor] = {}
        self._local_parameters: Dict[str, torch.Tensor] = {}
        # pseudo-gradients: views into one flat buffer per (dtype, device)
        self._grads: Dict[str, torch.Tensor] = {}
        self._flat_grads: List[torch.Tensor] = []

        bdev = self._backup_device or torch.device("cpu")
        for name, p in self._model_fragment.named_parameters():
            self._names.append(name)
            self._params.append(p)
            local = _local_view(p.data)
            t = torch.empty(tuple(local.shape), dtype=local.dtype, device=bdev)
            if self._pin_memory and t.device.type == "cpu" and torch.cuda.is_available():
                t = t.pin_memory()
            self.original_parameters[name] = t
        # persistent pseudo-gradient buffers in NVLink-symmetric memory (zero-copy / in-switch all-reduce)
        self._symm_flat: Dict[Tuple[torch.dtype, torch.device], torch.Tensor] = {}
        # Native fast path (see _try_flat_mode): the fragment is ONE flat buffer end to end
        self._flat_param: Optional[torch.Tensor] = None
        self._flat_orig: Optional[torch.Tensor] = None
        self._flat_grad: Optional[torch.Tensor] = None
        self._flat_mom: Optional[torch.Tensor] = None
        if not self._try_flat_mode():
            self._alloc_symmetric_buffers()

    # ------------------------------------------------------------------ flat fast path
    def _try_flat_mode(self) -> bool:
        """When the fragment's parameters are adjacent views of one CUDA buffer (``models.llama.FlatParams`` lays models
        out like that), the backup lives on the same GPU and the outer optimizer is momentum/Nesterov SGD, a sync is two
        launches over flat buffers instead of per-parameter copies + four passes:

        * ``prepare_sync``: ``allreduce_delta(flat_grad, flat_original, flat_param)`` -- ``original - local``, fp8
          quantisation, exchange, reduction and dequantisation in ONE kernel straight on symmetric memory;
        * ``perform_sync``: ``diloco_outer`` -- outer SGD step, save of the new global weights and the alpha merge in
          ONE kernel (reference: set grads + ``outer_optimizer.step()`` + ``save_parameters`` + ``_merge_parameters``,
          local_sgd.py:339-384,445-475).

        The outer optimizer object then only supplies hyper-parameters (lr schedulers keep working); its momentum lives in
        ``self._flat_mom`` (fp32) and travels with heals under ``"outer_momentum"``.
        """
        if os.environ.get("TORCHFT_B200_DILOCO_FLAT", "1") == "0" or not self._params:
            return False
        opt = self._outer_optimizer
        if type(opt) is not optim.SGD or len(opt.param_groups) != 1:
            return False
        g = opt.param_groups[0]
        if g.get("weight_decay", 0) != 0 or g.get("dampening", 0) != 0 or g.get("maximize", False):
            return False
        ps = [p.data for p in self._params]
        dev, dt = ps[0].device, ps[0].dtype
        if dev.type != "cuda" or dt not in (torch.float32, torch.bfloat16, torch.float16):
            return False
        if self._backup_device is None or torch.device(self._backup_device).type != "cuda":
            return False
        if any(_is_dtensor(p) or p.device != dev or p.dtype != dt or not p.is_contiguous() for p in ps):
            return False
        if {id(q) for q in g["params"]} != {id(q) for q in self._params}:
            return False
        es = ps[0].element_size()
        store = ps[0].untyped_storage()
        if any(p.untyped_storage().data_ptr() != store.data_ptr() for p in ps):
            return False
        order = sorted(range(len(ps)), key=lambda i: ps[i].data_ptr())
        lo = ps[order[0]].data_ptr()
        end = lo
        for i in order:
            if ps[i].data_ptr() < end or ps[i].data_ptr() - end > 4096 * es:  # overlapping or far apart: not one flat buffer
                return False
            end = ps[i].data_ptr() + ps[i].numel() * es
        if lo % 16:
            return False
        span = ((end - lo) // es + 7) // 8 * 8
        if (lo - store.data_ptr()) + span * es > store.nbytes():
            span = (end - lo) // es
        if not self._span_is_own(lo, lo + span * es):
            return False
        alloc = getattr(self._manager, "alloc_symmetric", None)
        if alloc is None or not self._manager.supports_fused_delta():
            return False
        try:
            buf = alloc(f"diloco_f{self._fragment_id}_flat", span * es)
            if self.should_quantize:  # scratch for the Q8G wire format: the whole fragment in one launch
                # whole fragment in wire format (fp32 scale + 512 e4m3 bytes per group, padded to a multiple of 8 groups)
                # + this rank's reduced slice (at most half of it again, at world 2)
                alloc(f"diloco_f{self._fragment_id}_q8", (span * 516 // 512 + 16 * 516 + 4096) * 3 // 2 + 8192)
        except Exception:  # noqa: BLE001 - group already configured etc.
            logger.exception("flat DiLoCo path unavailable (symmetric memory); using the generic path")
            return False
        if not isinstance(buf, torch.Tensor) or buf.device != dev:
            return False
        self._flat_param = torch.empty(0, dtype=dt, device=dev).set_(store, (lo - store.data_ptr()) // es, (span,))
        self._flat_grad = buf.view(dt)[:span]
        self._flat_grad.zero_()
        self._flat_orig = torch.empty(span, dtype=dt, device=dev)
        self._flat_mom = torch.zeros(span, dtype=torch.float32, device=dev)
        for name, p in zip(self._names, self._params):
            off = (p.data.data_ptr() - lo) // es
            self.original_parameters[name] = self._flat_orig[off: off + p.numel()].view(p.shape)
        return True

    def _span_is_own(self, lo: int, hi: int) -> bool:
        """True when the bytes ``[lo, hi)`` hold no weight of the inner optimizer outside this fragment. The flat path
        applies the outer step to its whole span, gaps and rounded tail included, so a weight of another fragment (or
        of none) lying there would be moved by this fragment's sync."""
        mine = {id(p) for p in self._params}
        for group in self._local_optimizer.param_groups:
            for q in group["params"]:
                t = _local_view(q.data)
                start = t.data_ptr()
                if id(q) not in mine and t.numel() and start < hi and lo < start + t.numel() * t.element_size():
                    return False
        return True

    def _group_sizes(self) -> Dict[Tuple[torch.dtype, torch.device], List[int]]:
        groups: Dict[Tuple[torch.dtype, torch.device], List[int]] = {}
        for i, p in enumerate(self._params):
            lp = _local_view(p.data)
            groups.setdefault((lp.dtype, lp.device), []).append(i)
        return groups

    def _alloc_symmetric_buffers(self) -> None:
        """When the manager's process group owns peer-visible memory (ProcessGroupB200), place the flat
        pseudo-gradient buffer there ONCE: every sync then reduces it in place (P2P or NVLS kernel)
        instead of bouncing through the staging buffer, and nothing is allocated per sync. Must run
        before the first quorum (segments are exchanged at configure time); replicas construct DiLoCo
        identically, so names and sizes match."""
        alloc = getattr(self._manager, "alloc_symmetric", None)
        if alloc is None:
            return
        for gi, ((dt, dev), idxs) in enumerate(self._group_sizes().items()):
            if dev.type != "cuda":
                continue
            total = sum((_local_view(self._params[i].data).numel() + 7) // 8 * 8 for i in idxs)
            try:
                buf = alloc(f"diloco_f{self._fragment_id}_g{gi}", total * torch.empty(0, dtype=dt).element_size())
            except Exception:  # noqa: BLE001 - e.g. group already configured: fall back to plain buffers
                logger.exception("symmetric pseudo-gradient buffer unavailable; using the staged path")
                continue
            if isinstance(buf, torch.Tensor) and buf.device == dev:
                flat = buf.view(dt)[:total]
                flat.zero_()  # alignment padding must stay finite (fp8 groups share a scale)
                self._symm_flat[(dt, dev)] = flat

    # --------------------------------------------------------------- heal hooks
    def register_state_dict_fn(self) -> None:
        """The backup weights and the outer optimizer must reach a healing replica too."""
        key = f"StreamingDiLoCoFragment_{self._fragment_id}"

        def load_fn(state_dict: Dict[str, Dict[str, torch.Tensor]]) -> None:
            for name, value in state_dict["original_parameters"].items():
                if name in self.original_parameters:
                    self.original_parameters[name].copy_(value)
            self._outer_optimizer.load_state_dict(state_dict["outer_optimizer"])
            if self._flat_mom is not None and "outer_momentum" in state_dict:
                self._flat_mom.copy_(state_dict["outer_momentum"])

        def save_fn() -> Dict[str, Dict[str, torch.Tensor]]:
            out = {
                "outer_optimizer": self._outer_optimizer.state_dict(),
                "original_parameters": {n: extract_local_tensor(t) for n, t in self.original_parameters.items()},
            }
            if self._flat_mom is not None:
                out["outer_momentum"] = self._flat_mom
            return out

        self._manager.register_state_dict_fn(key, load_fn, save_fn)

    # ------------------------------------------------------------ param copies
    @torch.profiler.record_function("torchft::local_sgd::save_parameters")
    def save_parameters(self) -> None:
        if self._flat_orig is not None:
            with torch.no_grad():
                self._flat_orig.copy_(self._flat_param)
            return
        with torch.no_grad():
            for name, p in zip(self._names, self._params):
                self.original_parameters[name].copy_(_local_view(p.data), non_blocking=True)

    def _save_local_parameters(self) -> None:
        with torch.no_grad():
            for name, p in zip(self._names, self._params):
                self._local_parameters[name] = extract_local_tensor(p.data)

    @torch.profiler.record_function("torchft::local_sgd::restore_parameters")
    def restore_parameters(self) -> None:
        if self._flat_orig is not None:
            with torch.no_grad():
                self._flat_param.copy_(self._flat_orig)
            return
        with torch.no_grad():
            for name, p in zip(self._names, self._params):
                _assign(p, self.original_parameters[name], non_blocking=False)

    def _clear_local_parameters(self) -> None:
        self._local_parameters = {}

    def _merge_parameters(self) -> None:
        with torch.no_grad():
            for name, p in zip(self._names, self._params):
                _local_view(p.data).lerp_(self._local_parameters[name], self._fragment_update_alpha)

    # ---------------------------------------------------------- pseudo-gradients
    def _launch_pseudograd_allreduce(self) -> None:
        """pseudo-gradient = original - local, averaged across replicas.

        One flat buffer per (dtype, device); messages are contiguous slices of at
        most ``bucket_cap_mb`` bytes when bucketization is on, else one slice per
        parameter. ``Manager.allreduce_delta`` fuses subtraction (+ fp8 quantisation)
        into the collective on ProcessGroupB200.
        """
        self._grads = {}
        self._flat_grads = []
        if self._flat_grad is not None:
            assert self._flat_orig is not None and self._flat_param is not None
            self._allreduce_work.append(self._manager.allreduce_delta(
                self._flat_grad, self._flat_orig, self._flat_param, should_quantize=self.should_quantize))
            return
        groups = self._group_sizes()
        locals_ = [_local_view(p.data) for p in self._params]
        fused = self.should_quantize and self._manager.supports_fused_delta()
        for (dt, dev), idxs in groups.items():
            sizes = [(locals_[i].numel() + 7) // 8 * 8 for i in idxs]  # 16 B aligned slices
            total = sum(sizes)
            # flat_grad starts out holding the ORIGINAL weights on the fused path (the kernel
            # computes original - local on the fly and overwrites it with the averaged result)
            flat_grad = self._symm_flat.get((dt, dev))
            if flat_grad is None or flat_grad.numel() != total:
                flat_grad = torch.zeros(total, dtype=dt, device=dev)
            flat_local = torch.zeros(total, dtype=dt, device=dev) if fused else None
            bounds: List[Tuple[int, int]] = []
            off = 0
            for i, sz in zip(idxs, sizes):
                n = locals_[i].numel()
                name = self._names[i]
                gview = flat_grad[off : off + n].view(locals_[i].shape)
                if fused:
                    gview.copy_(self.original_parameters[name], non_blocking=True)
                    flat_local[off : off + n].copy_(locals_[i].reshape(-1))
                else:
                    torch.sub(self.original_parameters[name].to(dev, non_blocking=True), locals_[i], out=gview)
                self._grads[name] = gview
                bounds.append((off, off + sz))
                off += sz
            self._flat_grads.append(flat_grad)
            if self.use_bucketization:
                cap = max(8, self.bucket_cap_mb // flat_grad.element_size() // 8 * 8)
                slices = [(lo, min(lo + cap, total)) for lo in range(0, total, cap)]
            else:
                slices = bounds
            for lo, hi in slices:
                if fused:
                    w = self._manager.allreduce_delta(flat_grad[lo:hi], flat_grad[lo:hi], flat_local[lo:hi],
                                                      should_quantize=True)
                else:
                    w = self._manager.allreduce(flat_grad[lo:hi], should_quantize=self.should_quantize)
                self._allreduce_work.append(w)

    def _set_grads(self) -> None:
        with torch.no_grad():
            for name, p in zip(self._names, self._params):
                g = self._grads.pop(name)
                if _is_dtensor(p):
                    p.grad = DTensor.from_local(g, p.device_mesh, p.placements, shape=p.shape, stride=p.stride())
                else:
                    p.grad = g

    # ------------------------------------------------------------------ schedule
    @torch.profiler.record_function("torchft::local_sgd::wait")
    def wait(self) -> None:
        """Block until the previously launched pseudo-gradient all-reduce has finished."""
        if not self._allreduce_work:
            return
        if self._stream is not None:
            assert self._stop_event is not None
            self._stop_event.synchronize()
            self._stop_event = None
        self._allreduce_work = []

    @torch.profiler.record_function("torchft::local_sgd::prepare_sync")
    def prepare_sync(self) -> None:
        """Compute pseudo-gradients and START averaging them (does not wait)."""
        assert len(self._allreduce_work) == 0
        if self._stream is not None:
            self._stream.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(self._stream) if self._stream is not None else nullcontext():
            self._launch_pseudograd_allreduce()
            if self._stream is not None:
                # a fused collective reads the weights on the process group's own stream: wait for it on this one
                for w in self._allreduce_work:
                    if not isinstance(w, DummyWork):  # a latched error: nothing was launched
                        w.block_current_stream()
                self._read_event = self._stream.record_event()

    def fence_weight_writes(self) -> None:
        """Make the current stream wait until the launched pseudo-gradient no longer reads the live weights. Called
        before every inner optimizer step: with ``fragment_sync_delay >= 1`` that step would otherwise write weights
        the quantisation or the subtraction has not read yet, so the pseudo-gradient would hold part of an extra inner
        step, different on every replica and every run. Forward and backward still run beside the all-reduce."""
        if self._read_event is not None:
            torch.cuda.current_stream().wait_event(self._read_event)
            self._read_event = None

    @torch.profiler.record_function("torchft::local_sgd::perform_sync")
    def perform_sync(self) -> bool:
        """Wait for the averaged pseudo-gradients, then commit: outer step, save, merge."""
        assert len(self._allreduce_work) > 0, "prepare_sync must run before perform_sync"
        with torch.cuda.stream(self._stream) if self._stream is not None else nullcontext():
            for w in self._allreduce_work:
                w.wait()
            if self._stream is not None:
                self._stop_event = torch.cuda.Event()
                self._stop_event.record()
        self.wait()

        if self._flat_grad is not None:
            return self._perform_sync_flat()

        self._save_local_parameters()  # needed for the alpha merge
        self.restore_parameters()      # back to the last global weights
        should_commit = self._manager.should_commit()
        if should_commit:
            self._set_grads()
            self._outer_optimizer.step()
            self.save_parameters()
            self._merge_parameters()
        self._outer_optimizer.zero_grad()
        self._clear_local_parameters()
        self._grads = {}
        self._flat_grads = []
        return should_commit


    def _perform_sync_flat(self) -> bool:
        """Commit decision, then ONE kernel: outer step on the last global weights, save them, merge with local."""
        from torchft_b200.ops import _native

        assert self._flat_param is not None and self._flat_orig is not None and self._flat_mom is not None
        t0 = _trace("   all-reduce waited", time.perf_counter())
        should_commit = self._manager.should_commit()
        t0 = _trace("   should_commit", t0)
        with torch.no_grad():
            if should_commit:
                g = self._outer_optimizer.param_groups[0]
                _native.load().diloco_outer(
                    self._flat_param.data_ptr(), self._flat_orig.data_ptr(), self._flat_grad.data_ptr(), self._flat_mom.data_ptr(),
                    self._flat_param.numel(), _native.dtype_code(self._flat_param), float(g["lr"]), float(g.get("momentum", 0.0)),
                    bool(g.get("nesterov", False)), float(self._fragment_update_alpha), 0, _native.stream_ptr())
            else:
                self._flat_param.copy_(self._flat_orig)  # the window is discarded: back to the last global weights
        return should_commit


class DiLoCo:
    """DiLoCo / Streaming DiLoCo (https://arxiv.org/abs/2311.08105, https://arxiv.org/abs/2501.18512).

    Replicas train independently with ``inner_optimizer``; every ``sync_every`` inner
    steps the averaged pseudo-gradient (last global weights minus current local
    weights) is applied by ``outer_optimizer``. With several ``model_fragments`` one
    fragment syncs every ``sync_every / n_fragments`` steps. A failed sync resets the
    fragment to its last global weights and retries at the next window.

    Requires ``Manager(use_async_quorum=False)``.
    """

    def __init__(self, manager: Manager, model_fragments: List[nn.Module], inner_optimizer: optim.Optimizer,
                 outer_optimizer: optim.Optimizer | List[optim.Optimizer], sync_every: int,
                 backup_device: Optional[torch.device] = None, pin_memory: bool = True,
                 use_bucketization: bool = False, bucket_cap_mb: Optional[int] = None, should_quantize: bool = False,
                 fragment_sync_delay: int = 0, fragment_update_alpha: float = 0.0) -> None:
        n = len(model_fragments)
        if isinstance(outer_optimizer, list):
            assert len(outer_optimizer) == n, "The number of outer optimizers must match the number of model fragments"
        if manager._use_async_quorum:
            raise ValueError("Using DiLoCo require synchronous quorum to be enabled. "
                             "Ensure that the manager is initialized with use_async_quorum=False")
        if sync_every < n:
            raise ValueError("Only 1 fragment can be syncrhonized at a time")
        if sync_every % n != 0:
            raise ValueError("sync_every must divide the number of fragments")
        self._sync_every = sync_every // n
        if fragment_sync_delay >= self._sync_every:
            raise ValueError("Fragment must be synced before it is reduced another time")
        if fragment_update_alpha < 0 or fragment_update_alpha > 1:
            raise ValueError("fragment_update_alpha must be between 0 and 1")

        self._manager = manager
        self._local_step = 0
        self._fragment_sync_delay = fragment_sync_delay
        self._hooks: List[RemovableHandle] = []
        self._local_optimizer = inner_optimizer
        self._fragments = [
            _StreamingDiLoCoFragment(
                manager, frag, i, math.floor((sync_every / n) * (i + 1)), inner_optimizer,
                outer_optimizer[i] if isinstance(outer_optimizer, list) else outer_optimizer,
                sync_every, backup_device, pin_memory, use_bucketization, bucket_cap_mb, should_quantize,
                fragment_sync_delay, fragment_update_alpha)
            for i, frag in enumerate(model_fragments)
        ]
        # step 0 must already have a valid global copy to fall back to
        self._save_parameters()
        for f in self._fragments:
            f.register_state_dict_fn()

    def _save_parameters(self) -> None:
        for f in self._fragments:
            f.save_parameters()

    def _restore_parameters(self) -> None:
        for f in self._fragments:
            f.restore_parameters()

    def __enter__(self) -> "DiLoCo":
        self._hooks.append(self._local_optimizer.register_step_pre_hook(self._step_pre_hook))
        self._hooks.append(self._local_optimizer.register_step_post_hook(self._step_post_hook))
        return self

    def __exit__(self, exc_type: Optional[Type[BaseException]], exc_value: Optional[BaseException],
                 traceback: Optional[TracebackType]) -> bool:
        for h in self._hooks:
            h.remove()
        self._hooks.clear()
        return False

    def _step_pre_hook(self, _optim: optim.Optimizer, _args: Tuple[Any, ...], _kwargs: Dict[str, Any]) -> None:
        self._manager.disallow_state_dict_read()
        for f in self._fragments:
            f.fence_weight_writes()

    def _wait(self) -> None:
        for f in self._fragments:
            f.wait()

    def _current_fragment(self) -> int:
        # derived from the COMMITTED step so every replica picks the same fragment
        return self._manager.current_step() % len(self._fragments)

    def _step_post_hook(self, _optim: optim.Optimizer, _args: Tuple[Any, ...], _kwargs: Dict[str, Any]) -> None:
        self._manager.allow_state_dict_read()
        self._local_step += 1

        t0 = _trace("inner step drained", time.perf_counter()) if self._local_step >= self._sync_every - self._fragment_sync_delay else 0.0
        if self._local_step == self._sync_every - self._fragment_sync_delay:
            # sync quorum: blocks, heals eagerly; every replica then prepares the SAME fragment
            self._manager.start_quorum()
            t0 = _trace("start_quorum (synchronous)", t0)
            frag = self._current_fragment()
            logger.info(f"Preparing fragment={frag} step={self._local_step}")
            self._fragments[frag].prepare_sync()
            t0 = _trace("prepare_sync (pseudo-gradient all-reduce enqueued + drained)", t0)

        if self._local_step < self._sync_every:
            return
        assert self._local_step == self._sync_every, f"{self._local_step=} should never exceed {self._sync_every=}"
        frag = self._current_fragment()
        logger.info(f"Syncing fragment={frag} step={self._local_step} manager_step={self._manager.current_step()}")
        self._fragments[frag].perform_sync()
        _trace("perform_sync (wait + should_commit + outer step)", t0)
        # on failure the parameters were reset to the last global copy; the window is retried
        self._local_step = 0
