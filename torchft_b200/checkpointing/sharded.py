"""Sharded durable checkpoints of FT-ZeRO-1: one file per (update count, quorum size, quorum rank).

Under FT-ZeRO-1 no replica holds the whole optimizer state, so every replica writes the slices it is the primary holder
of (see :meth:`~torchft_b200.parallel.zero1.Zero1Optimizer.save`); the files of one quorum tile the flat parameter
vector. This module owns the file format, the background writer and the ranged reader.

File ``z1_step_{T}.w{W}.r{r}.bin``::

    b"TFTZ1CKP" | u64 header bytes (little endian) | JSON header | zero pad to 16 bytes | payload

The payload holds four arrays over the ``elements`` written elements, back to back: ``param`` (bf16), ``master``,
``m`` and ``v`` (fp32; bf16 when the header says ``"moments": "bf16"``, a file without the key has fp32 moments), at the
byte offsets ``sections`` gives relative to the payload start. A file written with an EMA of the weights has
``"ema": {"decay": d}`` in its header and a fifth array ``ema`` of the moments' type behind ``v``. Each written range
``[lo, hi)`` of the flat vector is stored at element offset ``off`` of every array (``ranges``: ``[lo, hi, off]``).
Ranges are multiples of 8 elements, so every array and every range in it starts 16-byte aligned. The payload is read
with ranged ``pread`` calls only, never loaded whole.
"""

from __future__ import annotations

import json
import logging
import os
import re
import struct
import time
from typing import Any, Dict, List, Optional, Sequence, Tuple

import torch

from torchft_b200.checkpointing.durable import BackgroundWriter, atomic_write, prune_steps

logger = logging.getLogger(__name__)

__all__ = ["FORMAT_VERSION", "file_name", "sections", "moment_size", "file_dtype", "payload_bytes", "encode_header", "read_header", "scan", "check_compatible",
           "ShardedWriter", "RangedReader"]

FORMAT_VERSION = 1
MAGIC = b"TFTZ1CKP"
_NAME = re.compile(r"^z1_step_(\d+)\.w(\d+)\.r(\d+)\.bin$")
_ITEM = {"param": 2, "master": 4, "m": 4, "v": 4}


def file_name(step: int, world: int, rank: int) -> str:
    return f"z1_step_{step}.w{world}.r{rank}.bin"


def sections(elements: int, moment_size: int = 4, ema: bool = False) -> Dict[str, int]:
    """Byte offset of each array in the payload of a file holding ``elements`` elements: 14 bytes each with fp32
    moments, 10 with bf16 moments (``moment_size`` 2), and ``moment_size`` more for the ``ema`` section."""
    out, at = {}, 0
    for name, size in _ITEM.items():
        out[name] = at
        at += (moment_size if name in ("m", "v") else size) * elements
    if ema:
        out["ema"] = at
    return out


def moment_size(header: Dict[str, Any]) -> int:
    """Bytes per element of ``m`` and ``v`` in the file ``header`` describes; raises ``ValueError`` for an unknown type."""
    kind = header.get("moments", "fp32")
    if kind not in ("fp32", "bf16"):
        raise ValueError(f"unknown moment type {kind!r}")
    return 2 if kind == "bf16" else 4


def file_dtype(header: Dict[str, Any], array: str) -> torch.dtype:
    """The dtype ``array`` is stored in."""
    if array in ("m", "v", "ema"):
        return torch.bfloat16 if moment_size(header) == 2 else torch.float32
    return torch.bfloat16 if array == "param" else torch.float32


def payload_bytes(header: Dict[str, Any]) -> int:
    return (6 + (3 if "ema" in header else 2) * moment_size(header)) * int(header["elements"])


def encode_header(header: Dict[str, Any]) -> bytes:
    """Magic, length, JSON and padding: the bytes in front of the payload (a multiple of 16)."""
    body = json.dumps(header, separators=(",", ":")).encode()
    raw = MAGIC + struct.pack("<Q", len(body)) + body
    return raw + b"\0" * (-len(raw) % 16)


def read_header(path: str) -> Optional[Dict[str, Any]]:
    """The header of ``path`` plus ``path`` and ``data`` (absolute payload offset), or ``None`` (logged) when the file
    is not a readable checkpoint: wrong magic, version or header, or shorter than its header says."""
    try:
        with open(path, "rb") as f:
            pre = f.read(16)
            if len(pre) != 16 or pre[:8] != MAGIC:
                raise ValueError("not a sharded checkpoint")
            (n,) = struct.unpack("<Q", pre[8:])
            body = f.read(n)
            if len(body) != n:
                raise ValueError("truncated header")
            h = json.loads(body.decode())
            if h.get("version") != FORMAT_VERSION:
                raise ValueError(f"format version {h.get('version')}, expected {FORMAT_VERSION}")
            data = 16 + n + (-(16 + n) % 16)
            elements = int(h["elements"])
            if sum(hi - lo for lo, hi, _ in h["ranges"]) != elements:
                raise ValueError("ranges do not add up to the element count")
            need = data + payload_bytes(h)
            size = os.fstat(f.fileno()).st_size
            if size < need:
                raise ValueError(f"truncated: {size} bytes, the header describes {need}")
    except Exception as e:  # noqa: BLE001 - a torn or foreign file is skipped
        logger.warning("skipping unreadable sharded checkpoint %s: %s", path, e)
        return None
    h["path"], h["data"] = path, data
    return h


def scan(directory: str) -> List[Dict[str, Any]]:
    """Headers of every readable checkpoint file in ``directory`` (sorted by step, world, rank)."""
    if not os.path.isdir(directory):
        return []
    named = []
    for name in os.listdir(directory):
        m = _NAME.match(name)
        if m:
            named.append((tuple(int(x) for x in m.groups()), name))
    out = []
    for _, name in sorted(named):
        h = read_header(os.path.join(directory, name))
        if h is not None:
            out.append(h)
    return out


def check_compatible(headers: Sequence[Dict[str, Any]], numel: int, units: Sequence[Tuple[int, int]]) -> None:
    """``ValueError`` when a checkpoint was written for another flat vector: another ``numel`` or other unit ranges
    (another model, or another ``optimizer_blocks``)."""
    want = [list(map(int, u)) for u in units]
    for h in headers:
        if int(h["numel"]) != numel or [list(map(int, u)) for u in h["units"]] != want:
            raise ValueError(f"checkpoint {h['path']} was written for numel={h['numel']} with {len(h['units'])} units; "
                             f"this optimizer has numel={numel} with {len(want)} units")


class ShardedWriter:
    """One replica's writer: a pinned staging buffer the snapshot copies land in, and a background thread that waits
    for the copies, writes the file atomically and keeps this writer's ``keep`` newest steps."""

    def __init__(self, directory: str, keep: int = 2) -> None:
        if keep < 1:
            raise ValueError("keep must be >= 1")
        self.directory = directory
        self.keep = keep
        self.stage: Optional[torch.Tensor] = None
        self._writer = BackgroundWriter("sharded checkpoint")
        self._written: Dict[int, List[str]] = {}
        os.makedirs(directory, exist_ok=True)

    def staging(self, nbytes: int) -> torch.Tensor:
        """The pinned staging buffer, grown to at least ``nbytes``. Call after :meth:`wait`: the last write is done."""
        if self.stage is None or self.stage.numel() < nbytes:
            self.stage = None  # free the old buffer first
            self.stage = torch.empty(nbytes, dtype=torch.uint8, pin_memory=True)
        return self.stage

    def submit(self, header: Dict[str, Any], copied: Any) -> str:
        """Write ``header`` and the payload it describes from staging once the event ``copied`` has fired."""
        path = os.path.join(self.directory, file_name(int(header["T"]), int(header["world"]), int(header["rank"])))
        self._writer.start(self._write, path, header, copied)
        return path

    def _write(self, path: str, header: Dict[str, Any], copied: Any) -> None:
        t0 = time.perf_counter()
        copied.synchronize()
        assert self.stage is not None
        payload = memoryview(self.stage.numpy())[: payload_bytes(header)]
        chunk = 256 << 20

        def write(f: Any) -> None:
            f.write(encode_header(header))
            for at in range(0, len(payload), chunk):
                f.write(payload[at:at + chunk])

        atomic_write(path, write)
        step = int(header["T"])
        self._written.setdefault(step, [])
        if path not in self._written[step]:
            self._written[step].append(path)
        prune_steps(self._written, self.keep)
        for gone in sorted(self._written)[: -self.keep]:
            del self._written[gone]
        logger.info("sharded checkpoint step %d written in %.2fs -> %s", step, time.perf_counter() - t0, path)

    def wait(self) -> None:
        """Block until the in-flight write is on disk; re-raises its error."""
        self._writer.wait()


class RangedReader:
    """Disk -> pinned bounce buffer -> H2D copy on ``stream``, double-buffered: ``pread`` fills one buffer while the
    other one's copy runs. :meth:`close` waits for the last copy and closes the files."""

    def __init__(self, stream: torch.cuda.Stream, chunk_bytes: int = 64 << 20) -> None:
        self.stream = stream
        self.chunk = chunk_bytes
        self._bufs = [torch.empty(chunk_bytes, dtype=torch.uint8, pin_memory=True) for _ in range(2)]
        self._views = [memoryview(b.numpy()) for b in self._bufs]
        self._events: List[Optional[torch.cuda.Event]] = [None, None]
        self._next = 0
        self._fds: Dict[str, int] = {}
        self.bytes_read = 0

    def read(self, header: Dict[str, Any], array: str, elem_off: int, dst: torch.Tensor) -> None:
        """``dst`` (contiguous, device) <- elements ``[elem_off, elem_off + dst.numel())`` of ``array`` in the file."""
        path = header["path"]
        fd = self._fds.get(path)
        if fd is None:
            fd = self._fds[path] = os.open(path, os.O_RDONLY)
        assert dst.dtype == file_dtype(header, array), (array, dst.dtype)
        size = dst.element_size()
        pos = int(header["data"]) + int(header["sections"][array]) + elem_off * size
        out = dst.view(torch.uint8)
        n = out.numel()
        done = 0
        while done < n:
            i, self._next = self._next, self._next ^ 1
            if self._events[i] is not None:
                self._events[i].synchronize()  # the copy out of this buffer has finished
            c = min(self.chunk, n - done)
            got = 0
            while got < c:
                r = os.preadv(fd, [self._views[i][got:c]], pos + done + got)
                if r <= 0:
                    raise IOError(f"{path}: short read at byte {pos + done + got}")
                got += r
            with torch.cuda.stream(self.stream):
                out[done:done + c].copy_(self._bufs[i][:c], non_blocking=True)
                self._events[i] = self.stream.record_event()
            done += c
        self.bytes_read += n

    def close(self) -> None:
        for ev in self._events:
            if ev is not None:
                ev.synchronize()
        for fd in self._fds.values():
            os.close(fd)
        self._fds.clear()
