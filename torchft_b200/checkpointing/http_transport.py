"""HTTP live-checkpoint transport (TCP fallback / CPU path).

Behavioural parity with the reference's default heal transport
(upstream torchft/checkpointing/http_transport.py:38-298): the source
stages its state_dict to host memory on a side stream, serves it from a
threaded HTTP server while the checkpoint is "allowed", rejects requests for a
different step with HTTP 400, and blocks new requests again in
``disallow_checkpoint``. ``num_chunks > 0`` splits the pytree leaves round-robin
into that many independently fetched streams. On a single NVSwitch domain
prefer :class:`~torchft_b200.checkpointing.p2p_transport.P2PTransport`, which
never leaves HBM.
"""

from __future__ import annotations

import io
import logging
import pickle
import socket
import threading
import urllib.request
from concurrent.futures import ThreadPoolExecutor
from contextlib import nullcontext
from datetime import timedelta
from http.server import BaseHTTPRequestHandler, ThreadingHTTPServer
from typing import Any, Generic, List, Optional, TypeVar

import torch
from torch.utils import _pytree as pytree

from torchft_b200.checkpointing._rwlock import RWLock
from torchft_b200.checkpointing._serialization import streaming_load, streaming_save
from torchft_b200.checkpointing.transport import CheckpointTransport

logger = logging.getLogger(__name__)


from torchft_b200.checkpointing.transport import advertise_host as _advertise_host  # noqa: E402

T = TypeVar("T")


class _Server(ThreadingHTTPServer):
    address_family = socket.AF_INET6
    request_queue_size = 1024
    daemon_threads = True

    def server_bind(self) -> None:
        # dual-stack so both 127.0.0.1 and [::1] clients work
        try:
            self.socket.setsockopt(socket.IPPROTO_IPV6, socket.IPV6_V6ONLY, 0)
        except OSError:
            pass
        super().server_bind()


def _to_cpu(obj: Any, pin: bool) -> Any:
    def one(x: Any) -> Any:
        if isinstance(x, torch.Tensor) and x.device.type != "cpu":
            out = torch.empty(x.shape, dtype=x.dtype, device="cpu", pin_memory=pin)
            out.copy_(x, non_blocking=True)
            return out
        return x

    return pytree.tree_map(one, obj)


class HTTPTransport(CheckpointTransport[T], Generic[T]):
    """Heal over HTTP (the reference's default transport, checkpointing/http_transport.py:38-298).

    ``send_checkpoint`` stages the state on the host and releases a write lock; GET ``/checkpoint/<step>/full``
    (or ``/metadata`` + ``/<chunk>`` when ``num_chunks > 0``, fetched in parallel) streams it socket-to-tensor;
    a request for another step gets 400; ``disallow_checkpoint`` re-takes the lock before the optimizer mutates state.
    """

    def __init__(self, timeout: timedelta, num_chunks: int = 0) -> None:
        self._timeout = timeout
        self._num_chunks = num_chunks
        self._lock = RWLock(timeout=timeout.total_seconds())
        self._lock.w_acquire()  # nothing to serve yet
        self._allowed = False
        self._step = -1
        self._state: Optional[Any] = None
        self._stream = torch.cuda.Stream() if torch.cuda.is_available() else None
        transport = self

        class Handler(BaseHTTPRequestHandler):
            protocol_version = "HTTP/1.1"

            def log_message(self, fmt: str, *args: Any) -> None:  # quiet
                logger.debug("http_transport: " + fmt, *args)

            def _fail(self, code: int, msg: str) -> None:
                body = msg.encode()
                self.send_response(code)
                self.send_header("Content-Type", "text/plain")
                self.send_header("Content-Length", str(len(body)))
                self.end_headers()
                self.wfile.write(body)

            def do_GET(self) -> None:  # noqa: N802
                parts = self.path.strip("/").split("/")
                if len(parts) != 3 or parts[0] != "checkpoint":
                    return self._fail(404, f"unknown path {self.path}")
                try:
                    step = int(parts[1])
                except ValueError:
                    return self._fail(400, "bad step")
                try:
                    with transport._lock.r_lock():
                        if step != transport._step:
                            return self._fail(400, f"invalid checkpoint requested: serving {transport._step} but got {step}")
                        # Stream straight from the staged tensors into the socket: no whole-payload buffer on
                        # the sender (a 16 GB state would otherwise exist three times). The body is delimited
                        # by connection close, so a failure mid-stream surfaces as a truncated read.
                        self.send_response(200)
                        self.send_header("Content-Type", "application/octet-stream")
                        self.send_header("Connection", "close")
                        self.end_headers()
                        self.close_connection = True
                        out = io.BufferedWriter(self.wfile, buffer_size=4 << 20)  # type: ignore[arg-type]
                        try:
                            transport._write_payload(parts[2], out)
                            out.flush()
                        finally:
                            out.detach()  # the wrapper must not close the handler's wfile when it is collected
                except TimeoutError as e:
                    self._fail(503, f"checkpoint not available: {e}")
                except (BrokenPipeError, ConnectionResetError):
                    pass
                except Exception as e:  # pragma: no cover - defensive
                    logger.exception("http_transport handler failed")
                    try:
                        self._fail(500, str(e))
                    except Exception:
                        pass

        self._server = _Server(("::", 0), Handler)
        self._thread = threading.Thread(target=self._server.serve_forever, name="tft_http_ckpt", daemon=True)
        self._thread.start()

    # ------------------------------------------------------------ server side
    def _write_payload(self, what: str, out: Any) -> None:
        state = self._state
        if what == "full":
            streaming_save(state, out)
            return
        leaves, spec = pytree.tree_flatten(state)
        if what == "metadata":
            pickle.dump({"treespec": spec, "num_leaves": len(leaves), "num_chunks": self._num_chunks}, out)
        else:
            streaming_save(leaves[int(what) :: max(self._num_chunks, 1)], out)

    def address(self) -> str:
        port = self._server.socket.getsockname()[1]
        return f"http://{_advertise_host()}:{port}"

    def metadata(self) -> str:
        return f"{self.address()}/checkpoint/"

    def send_checkpoint(self, dst_ranks: List[int], step: int, state_dict: T, timeout: timedelta) -> None:
        ctx = torch.cuda.stream(self._stream) if self._stream is not None else nullcontext()
        with ctx:
            if self._stream is not None:
                self._stream.wait_stream(torch.cuda.current_stream())
            staged = _to_cpu(state_dict, pin=False)
            if self._stream is not None:
                self._stream.synchronize()
        self._state = staged
        self._step = step
        self.allow_checkpoint(step)

    def allow_checkpoint(self, step: int) -> None:
        self._step = step
        if not self._allowed:
            self._allowed = True
            self._lock.w_release()

    def disallow_checkpoint(self) -> None:
        if self._allowed:
            self._allowed = False
            self._lock.w_acquire()
            self._state = None

    # ------------------------------------------------------------ client side
    def _get(self, url: str, timeout: timedelta) -> bytes:
        with urllib.request.urlopen(url, timeout=timeout.total_seconds()) as r:
            return r.read()

    def _load(self, url: str, timeout: timedelta) -> Any:
        """Deserialise while the bytes arrive (tensors are filled straight from the socket)."""
        with urllib.request.urlopen(url, timeout=timeout.total_seconds()) as r:
            return streaming_load(io.BufferedReader(r, buffer_size=4 << 20))  # type: ignore[arg-type]

    def recv_checkpoint(self, src_rank: int, metadata: str, step: int, timeout: timedelta) -> T:
        base = f"{metadata}{step}"
        try:
            if self._num_chunks <= 0:
                return self._load(f"{base}/full", timeout)
            meta = pickle.loads(self._get(f"{base}/metadata", timeout))
            n = max(int(meta["num_chunks"]), 1)
            with ThreadPoolExecutor(max_workers=n, thread_name_prefix="tft_http_recv") as ex:
                parts = list(ex.map(lambda i: self._load(f"{base}/{i}", timeout), range(n)))
            leaves: List[Any] = [None] * int(meta["num_leaves"])
            for i, chunk in enumerate(parts):
                leaves[i::n] = chunk
            return pytree.tree_unflatten(leaves, meta["treespec"])
        except urllib.error.HTTPError as e:  # type: ignore[attr-defined]
            raise RuntimeError(f"checkpoint fetch from rank {src_rank} failed: {e.code} {e.read().decode(errors='replace')}") from e
        except (socket.timeout, TimeoutError) as e:
            raise TimeoutError(f"checkpoint fetch from rank {src_rank} timed out: {e}") from e

    def shutdown(self, wait: bool = True) -> None:
        self._server.shutdown()
        self._server.server_close()
        if wait:
            self._thread.join(timeout=5)
