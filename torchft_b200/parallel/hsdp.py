"""Fault-tolerant HSDP trainer: FSDP2 shards INSIDE a replica group, torchft_b200 ACROSS groups.

BASELINE.json config 2 ("4 replica groups x 2-GPU FSDP shards"), wired the way the reference composes it
(upstream torchft/fsdp_test.py:57-72, README.md:62-69): ``fully_shard`` over the group's own mesh,
``set_all_reduce_hook`` so every reduce-scattered gradient shard is averaged across replica groups through a
``ManagedProcessGroup`` (-> ``Manager.allreduce`` -> the fused NVLink all-reduce kernel on ``ProcessGroupB200``, with
the 1/num_participants scale and the zero contribution of healing groups inside the kernel), one Manager per rank,
one ManagerServer per group, ``should_commit`` as the AND-barrier over the group's ranks.

All ranks of ALL groups may live in one ``torchrun`` world (how ``bench.py --shards S`` is launched): rank ``r`` is
shard ``r % S`` of group ``r // S``; intra-group collectives (FSDP all-gather / reduce-scatter) run on plain NCCL
sub-groups, which is outside the fault-tolerance scope exactly as in the reference.
"""

from __future__ import annotations

import os
from datetime import timedelta
from typing import Any, Dict, Optional

import torch
import torch.distributed as dist
from torch.distributed import TCPStore


def _local(t: Any) -> Any:
    """The local shard of a DTensor (aliasing its storage), anything else unchanged."""
    return t.to_local() if hasattr(t, "to_local") else t


def fsdp_local_state(model: torch.nn.Module, optim: torch.optim.Optimizer) -> Dict[str, Any]:
    """Heal payload of ONE rank of an FSDP2-sharded model: its local parameter shards and its local optimizer-state
    shards, keyed by parameter name, as plain tensors that ALIAS the live storage. A healthy replica serves them to the
    same group rank of the healing replica group (the reference heals rank i from rank i: manager.py:700-716); an
    in-place transport (``P2PTransport``) on the healing side writes straight into the tensors this function returns
    there, so a heal is one ranged NVLink copy per shard and no re-sharding is involved (same shard layout on both sides:
    replica groups are congruent by construction)."""
    params, state = {}, {}
    for name, p in model.named_parameters():
        params[name] = _local(p.detach())
        st = optim.state.get(p)
        if st:
            state[name] = {k: _local(v.detach()) if isinstance(v, torch.Tensor) else v for k, v in st.items()}
    return {"params": params, "optim": state}


@torch.no_grad()
def load_fsdp_local_state(model: torch.nn.Module, optim: torch.optim.Optimizer, payload: Dict[str, Any]) -> None:
    """Install a payload of :func:`fsdp_local_state` (tensors that are already the live storage are left alone;
    optimizer state a fresh replica does not have yet is created with the parameter's own sharding)."""
    for name, p in model.named_parameters():
        src = payload["params"][name]
        dst = _local(p.detach())
        if src.shape != dst.shape:
            raise ValueError(f"shard of {name}: got {tuple(src.shape)}, this rank holds {tuple(dst.shape)} (different sharding?)")
        if src.data_ptr() != dst.data_ptr():
            dst.copy_(src)
        incoming = payload["optim"].get(name)
        if incoming is None:
            optim.state.pop(p, None)  # the source had not stepped this parameter yet
            continue
        st = optim.state[p]  # defaultdict: creates the entry on a fresh replica
        for k, v in incoming.items():
            if not isinstance(v, torch.Tensor):
                st[k] = v
                continue
            cur = st.get(k)
            if cur is None:
                if v.dim() > 0 and v.shape == dst.shape:
                    cur = torch.zeros_like(p, dtype=v.dtype)  # per-element state follows the parameter's sharding
                else:
                    cur = v.detach().clone()                  # scalars (AdamW's step counter) are plain tensors
                st[k] = cur
            tgt = _local(cur)
            if tgt.data_ptr() != v.data_ptr():
                tgt.copy_(v)


class SymmetricShardGrads:
    """FSDP2 reduce-scatter communicator (``FSDPModule.set_custom_reduce_scatter``) whose OUTPUT buffers -- the fp32
    gradient shards that FSDP2 then hands to the cross-replica all-reduce hook and finally installs as ``param.grad`` --
    are carved out of one NVLink-symmetric arena of ``ProcessGroupB200``. The cross-replica all-reduce of a shard is then
    the zero-copy in-place kernel over peer memory (same arena offset on every replica group: backward visits the FSDP
    groups in the same order everywhere) instead of staging 2 x 436 MB per block through the 256 MB bounce buffer.

    The arena is a bump allocator: ``begin_step()`` (before backward) rewinds it; it must hold one step's worth of
    gradient shards (they stay alive until the optimizer has consumed them). The reduce-scatter INPUT stays an ordinary
    allocation, and the reduce-scatter itself is the stock intra-group collective."""

    def __init__(self, arena: torch.Tensor) -> None:
        self._arena = arena  # uint8, symmetric
        self._off = 0
        self._want_output = False
        self.fallbacks = 0

    def begin_step(self) -> None:
        self._off = 0
        self._want_output = False

    def allocate(self, size: Any, *, dtype: torch.dtype, device: torch.device) -> torch.Tensor:
        # FSDP2 (foreach_reduce) allocates strictly input, output, input, output, ...
        is_output, self._want_output = self._want_output, not self._want_output
        if is_output:
            n = 1
            for d in size:
                n *= int(d)
            nbytes = n * torch.empty((), dtype=dtype).element_size()
            lo = (self._off + 255) // 256 * 256
            if lo + nbytes <= self._arena.numel():
                self._off = lo + nbytes
                return self._arena[lo:lo + nbytes].view(dtype).view(*[int(d) for d in size])
            self.fallbacks += 1  # arena too small (gradient accumulation over several backwards): staged path
        return torch.empty(*size, dtype=dtype, device=device)

    def __call__(self, output_tensor: torch.Tensor, input_tensor: torch.Tensor, group: dist.ProcessGroup, op: Any,
                 async_op: bool = False) -> Any:
        return dist.reduce_scatter_tensor(output=output_tensor, input=input_tensor, group=group, op=op, async_op=async_op)


class HSDPTrainer:
    """Llama over ``groups x shards`` GPUs.

    Args:
        model: config name in ``models.llama.CONFIGS``
        lighthouse_addr: address of a running Lighthouse
        shards: FSDP degree inside a replica group (the torchrun world is cut into consecutive blocks of this size)
        backend: ``"b200"`` (native cross-replica kernels) or ``"nccl"`` (reference-equivalent arm)
    """

    def __init__(self, model: str, lighthouse_addr: str, shards: int, backend: str = "b200", lr: float = 3e-4,
                 timeout: timedelta = timedelta(seconds=120), device: Optional[torch.device] = None, seed: int = 0,
                 replica_prefix: str = "hsdp") -> None:
        from torch.distributed.device_mesh import init_device_mesh
        from torch.distributed.fsdp import MixedPrecisionPolicy, fully_shard

        from torchft_b200 import ManagedProcessGroup, Manager, Optimizer
        from torchft_b200.models.llama import CONFIGS, Llama

        if CONFIGS[model].tie_embeddings:
            # the tied head writes the embedding's gradient during the forward, which FSDP2's sharded gradients and
            # reduce-scatter hooks do not provide for
            raise ValueError(f"HSDPTrainer does not train models with tied embeddings ({model}); use "
                             "FaultTolerantTrainer")

        assert dist.is_initialized(), "init the NCCL world first (torchrun)"
        rank, world = dist.get_rank(), dist.get_world_size()
        assert world % shards == 0
        self.groups, self.shards = world // shards, shards
        self.group, self.group_rank = rank // shards, rank % shards
        self.device = device if device is not None else torch.device("cuda", torch.cuda.current_device())
        self.cfg = CONFIGS[model]
        mesh = init_device_mesh("cuda", (self.groups, shards), mesh_dim_names=("replicate", "shard"))
        shard_mesh = mesh["shard"]
        shard_pg = shard_mesh.get_group()

        # the group's store: hosted by its shard rank 0, port shared over the (NCCL) shard group
        port = [0]
        if self.group_rank == 0:
            self._store = TCPStore("127.0.0.1", 0, is_master=True, wait_for_workers=False)
            port = [self._store.port]
        dist.broadcast_object_list(port, group=shard_pg, group_src=0)

        # fp32 master parameters sharded by FSDP2, bf16 compute copies, fp32 gradient reduction
        torch.manual_seed(seed)
        m = Llama(self.cfg, device=self.device, dtype=torch.float32)
        m.init_weights(seed)
        # cast_forward_inputs=False: the blocks' inputs are the bf16 residual stream and the fp32 RoPE table, which the
        # RoPE kernel reads as fp32 (the default would hand it a bf16 copy)
        mp = MixedPrecisionPolicy(param_dtype=torch.bfloat16, reduce_dtype=torch.float32, cast_forward_inputs=False)
        for blk in m.layers:
            fully_shard(blk, mesh=shard_mesh, mp_policy=mp)
        fully_shard(m, mesh=shard_mesh, mp_policy=mp)
        self.model = m

        if backend == "b200":
            from torchft_b200.parallel.process_group_b200 import ProcessGroupB200

            self.pg: Any = ProcessGroupB200(timeout=timeout, device=self.device)
            # one step's fp32 gradient shards live in symmetric memory (see SymmetricShardGrads); 256 B per FSDP group
            # of alignment slack
            shard_bytes = sum(-(-p.numel() // shards) for p in m.parameters()) * 4 + 256 * (len(m.layers) + 2) + (1 << 20)
            self._grad_arena: Optional[SymmetricShardGrads] = SymmetricShardGrads(self.pg.alloc_symmetric("hsdp_grads", shard_bytes))
        else:
            from torchft_b200.process_group import ProcessGroupNCCL

            self.pg = ProcessGroupNCCL(timeout=timeout)
            self._grad_arena = None
        self.manager = Manager(pg=self.pg, load_state_dict=None, state_dict=None, min_replica_size=self.groups,
                               timeout=timeout, quorum_timeout=timeout, connect_timeout=timeout, rank=self.group_rank,
                               world_size=shards, store_addr="127.0.0.1", store_port=int(port[0]),
                               lighthouse_addr=lighthouse_addr, replica_id=f"{replica_prefix}_{self.group}", init_sync=False)
        # heal: rank i of a joining group pulls the parameter and optimizer shards of rank i of a healthy group in place
        self.manager.register_state_dict_fn("hsdp", lambda sd: load_fsdp_local_state(self.model, self.inner, sd),
                                            lambda: fsdp_local_state(self.model, self.inner))
        replicate = ManagedProcessGroup(self.manager)

        def cross_replica(shard_grad: torch.Tensor) -> None:
            # FSDP2 hands over the reduce-scattered gradient shard of one parameter group, on its reduce stream
            replicate.allreduce([shard_grad], dist.ReduceOp.AVG).wait()

        for mod in m.modules():
            if hasattr(mod, "set_all_reduce_hook"):
                mod.set_all_reduce_hook(cross_replica)
                if self._grad_arena is not None:
                    mod.set_custom_reduce_scatter(self._grad_arena)
        self.inner = torch.optim.AdamW(m.parameters(), lr=lr, betas=(0.9, 0.95), weight_decay=0.1, fused=True)
        self.optim = Optimizer(self.manager, self.inner)
        self._tok: Optional[torch.Tensor] = None
        self._tgt: Optional[torch.Tensor] = None
        self._loss_host: Optional[torch.Tensor] = None
        self._loss_event: Optional[torch.cuda.Event] = None
        self.zero1 = False
        self.zopt = None

    def step_device(self, tokens: torch.Tensor, targets: torch.Tensor) -> torch.Tensor:
        self.optim.zero_grad(set_to_none=True)   # start_quorum (async)
        if self._grad_arena is not None:
            self._grad_arena.begin_step()        # last step's gradient shards are gone: rewind the symmetric arena
        loss = self.model(tokens, targets)
        loss.backward()                          # FSDP reduce-scatter + cross-replica hook per block, overlapped
        self.optim.step()                        # should_commit (AND over the group's ranks), then AdamW on the shards
        return loss

    def join(self) -> None:
        pass

    def _stage(self, tokens_cpu: torch.Tensor, targets_cpu: torch.Tensor) -> None:
        if self._tok is None or self._tok.shape != tokens_cpu.shape:
            self._tok = torch.empty(tokens_cpu.shape, dtype=torch.int64, device=self.device)
            self._tgt = torch.empty(tokens_cpu.shape, dtype=torch.int64, device=self.device)
        assert self._tgt is not None
        self._tok.copy_(tokens_cpu, non_blocking=True)
        self._tgt.copy_(targets_cpu, non_blocking=True)

    def step_async(self, tokens_cpu: torch.Tensor, targets_cpu: torch.Tensor) -> Optional[float]:
        prev = None
        if self._loss_event is not None:
            self._loss_event.synchronize()
            prev = float(self._loss_host[0])  # type: ignore[index]
        self._stage(tokens_cpu, targets_cpu)
        loss = self.step_device(self._tok, self._tgt)  # type: ignore[arg-type]
        if self._loss_host is None:
            self._loss_host = torch.empty(1, dtype=torch.float32).pin_memory()
            self._loss_event = torch.cuda.Event()
        self._loss_host.copy_(loss.detach().float().reshape(1), non_blocking=True)
        self._loss_event.record()  # type: ignore[union-attr]
        return prev

    def last_loss(self) -> Optional[float]:
        if self._loss_event is None:
            return None
        self._loss_event.synchronize()
        return float(self._loss_host[0])  # type: ignore[index]

    def shutdown(self) -> None:
        self.manager.shutdown(wait=False)
        self.pg.shutdown()
