"""Durable (on-disk) checkpoints next to the live peer-to-peer heal.

The reference deliberately stops at live recovery: "users must persist ``manager.state_dict()`` along with
model / optimizer / dataloader state" (``torchft/manager.py:158-159,967-977``, ``train_ddp.py:200-207``).
Live healing covers the loss of *some* replicas; a whole-job restart (all replicas gone, planned
maintenance, Lighthouse host lost) still needs a file. This helper packages the recipe so every script
does not re-invent it:

* **what**: ``{"user": state_dict_fn(), "torchft": manager.state_dict()}`` — exactly the payload a healing
  replica receives, so ``restore()`` can reuse the job's ``load_state_dict`` hook;
* **who**: replicas hold identical state after a commit, so only ONE of them writes — the participant with
  replica rank 0 (ties in multi-rank groups are broken by writing one file per group rank);
* **when**: ``maybe_save()`` right after a committed step, every ``every_n_steps``; the state is snapshotted
  to host memory synchronously (the optimizer is about to mutate it) and written by a background thread;
* **how**: temp file + ``os.replace`` (atomic on POSIX), newest ``keep`` files retained, a ``LATEST`` marker
  written last; a torn or truncated file is skipped by ``restore()``, which falls back to the previous one.

    ckpt = DurableCheckpointer(manager, state_dict=save_fn, load_state_dict=load_fn, directory="/ckpt/run1")
    ckpt.restore()                       # no-op on a fresh run
    for batch in data:
        optimizer.zero_grad(); loss(model(batch)).backward(); optimizer.step()
        ckpt.maybe_save()
"""

from __future__ import annotations

import logging
import os
import re
import threading
import time
from typing import Any, BinaryIO, Callable, Dict, List, Optional, Sequence

import torch
from torch.utils import _pytree as pytree

from torchft_b200.checkpointing._serialization import streaming_load, streaming_save

logger = logging.getLogger(__name__)

__all__ = ["DurableCheckpointer", "BackgroundWriter", "atomic_write", "prune_steps"]

_NAME = re.compile(r"^step_(\d+)\.rank_(\d+)\.pt$")


def _to_host(tree: Any) -> Any:
    """Deep copy with every tensor on the CPU (DTensors are saved as their local shards)."""

    def leaf(x: Any) -> Any:
        if isinstance(x, torch.Tensor):
            local = x.to_local() if hasattr(x, "to_local") else x
            return local.detach().to("cpu", copy=True)
        return x

    return pytree.tree_map(leaf, tree)


def atomic_write(path: str, write: Callable[[BinaryIO], None]) -> None:
    """Write ``path`` through a temporary file next to it, fsync it and ``os.replace`` it into place (atomic on POSIX):
    a reader sees the previous file or the complete new one, never a partial write under the final name."""
    tmp = f"{path}.tmp.{os.getpid()}"
    with open(tmp, "wb") as f:
        write(f)
        f.flush()
        os.fsync(f.fileno())
    os.replace(tmp, path)


def prune_steps(paths: Dict[int, Sequence[str]], keep: int) -> None:
    """Remove the files of every step but the ``keep`` newest (``paths[step]``: that step's files)."""
    for step in sorted(paths)[: -keep]:
        for path in paths[step]:
            try:
                os.remove(path)
            except OSError:
                pass


class BackgroundWriter:
    """At most one write in flight, on a daemon thread; an exception it raises is re-raised by the next :meth:`wait`
    (and so by the next :meth:`start`) instead of being lost."""

    def __init__(self, what: str) -> None:
        self._what = what
        self._thread: Optional[threading.Thread] = None
        self._error: Optional[BaseException] = None

    def start(self, fn: Callable[..., None], *args: Any) -> None:
        self.wait()
        self._thread = threading.Thread(target=self._run, args=(fn, args), name="tft_ckpt_writer", daemon=True)
        self._thread.start()

    def _run(self, fn: Callable[..., None], args: Any) -> None:
        try:
            fn(*args)
        except BaseException as e:  # noqa: BLE001 - reported on the next wait()
            self._error = e

    def wait(self) -> None:
        """Block until the in-flight write (if any) has finished; re-raises its error."""
        if self._thread is not None:
            self._thread.join()
            self._thread = None
        if self._error is not None:
            e, self._error = self._error, None
            raise RuntimeError(f"{self._what} write failed: {e}") from e


class DurableCheckpointer:
    """Periodic on-disk checkpoints of ``{user state, manager.state_dict()}`` written by ONE replica (see the module docstring).

    Args:
        manager: the job's :class:`~torchft_b200.Manager` (``current_step``, ``participating_rank``, ``state_dict``).
        state_dict / load_state_dict: the same hooks the Manager uses for live healing.
        directory: shared (or per-node) directory; files are ``step_<N>.rank_<group_rank>.pt``.
        every_n_steps: checkpoint cadence in committed steps; keep: how many files to retain per group rank.
    """

    def __init__(self, manager: Any, state_dict: Callable[[], Any], load_state_dict: Callable[[Any], None], directory: str,
                 every_n_steps: int = 100, keep: int = 2, group_rank: Optional[int] = None) -> None:
        if every_n_steps < 1 or keep < 1:
            raise ValueError("every_n_steps and keep must be >= 1")
        self._manager = manager
        self._state_dict = state_dict
        self._load_state_dict = load_state_dict
        self._dir = directory
        self._every = every_n_steps
        self._keep = keep
        self._group_rank = int(group_rank if group_rank is not None else getattr(manager, "_group_rank", 0))
        self._last_saved_step = -1
        self._writer = BackgroundWriter("durable checkpoint")
        os.makedirs(directory, exist_ok=True)

    # ------------------------------------------------------------------ save
    def _should_write(self) -> bool:
        """One writer per group rank: the participating replica with rank 0."""
        try:
            return self._manager.participating_rank() == 0
        except Exception:  # noqa: BLE001 - e.g. before the first quorum
            return False

    def maybe_save(self, force: bool = False) -> bool:
        """Call after ``optimizer.step()``. Returns True when a checkpoint write was started."""
        step = int(self._manager.current_step())
        if step == self._last_saved_step or step <= 0:
            return False
        if not force and step % self._every:
            return False
        if not self._should_write():
            return False
        self.wait()  # at most one write in flight; surfaces the previous write's error
        payload = {"user": _to_host(self._state_dict()), "torchft": dict(self._manager.state_dict())}
        self._last_saved_step = step
        self._writer.start(self._write, step, payload)
        return True

    def _path(self, step: int) -> str:
        return os.path.join(self._dir, f"step_{step}.rank_{self._group_rank}.pt")

    def _write(self, step: int, payload: Dict[str, Any]) -> None:
        t0 = time.perf_counter()
        final = self._path(step)
        atomic_write(final, lambda f: streaming_save(payload, f))
        marker = os.path.join(self._dir, f"LATEST.rank_{self._group_rank}")
        with open(marker + ".tmp", "w") as f:
            f.write(os.path.basename(final))
        os.replace(marker + ".tmp", marker)
        self._prune()
        logger.info("durable checkpoint step %d written in %.2fs -> %s", step, time.perf_counter() - t0, final)

    def _mine(self) -> List[int]:
        steps = []
        for name in os.listdir(self._dir):
            m = _NAME.match(name)
            if m and int(m.group(2)) == self._group_rank:
                steps.append(int(m.group(1)))
        return sorted(steps)

    def _prune(self) -> None:
        prune_steps({step: [self._path(step)] for step in self._mine()}, self._keep)

    def wait(self) -> None:
        """Block until the in-flight write (if any) is on disk; re-raises its error."""
        self._writer.wait()

    # --------------------------------------------------------------- restore
    def latest_step(self) -> Optional[int]:
        steps = self._mine()
        return steps[-1] if steps else None

    def restore(self) -> Optional[int]:
        """Load the newest readable checkpoint of this group rank; returns its step or None on a fresh run.

        Every replica that restarts restores the same file (shared filesystem) or its own copy; replicas
        that restore an OLDER step than a live peer are healed forward by the normal protocol at the first
        quorum, so a partially written newest checkpoint is harmless."""
        for step in reversed(self._mine()):
            path = self._path(step)
            try:
                with open(path, "rb") as f:
                    payload = streaming_load(f)
                user, meta = payload["user"], payload["torchft"]
            except Exception as e:  # noqa: BLE001 - torn file: try the previous one
                logger.warning("skipping unreadable checkpoint %s: %s", path, e)
                continue
            self._load_state_dict(user)
            self._manager.load_state_dict(meta)
            self._last_saved_step = int(meta.get("step", step))
            logger.info("restored durable checkpoint %s (step %s)", path, meta.get("step"))
            return int(meta.get("step", step))
        return None
