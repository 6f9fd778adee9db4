"""Prototype parameter server on reconfigurable process groups.

Parity: upstream torchft/parameter_server.py:30-194. A client GETs
``/new_session`` and receives ``{"session_id", "store_addr"}``; both sides then
configure a fresh 2-rank group (server = rank 0, client = rank 1) under that
store prefix and the server runs :meth:`forward` for the session. The Lighthouse
is not involved. Our server thread hands the session to a worker thread instead
of hijacking the HTTP handler thread, so a slow session cannot exhaust the
HTTP accept pool, and sessions are tracked for ``shutdown``.
"""

from __future__ import annotations

import json
import logging
import socket
import threading
import urllib.request
import uuid
from abc import ABC, abstractmethod
from http.server import BaseHTTPRequestHandler, ThreadingHTTPServer
from typing import Dict

from torch.distributed import TCPStore

from torchft_b200.process_group import ProcessGroup

logger = logging.getLogger(__name__)


def _advertise_host() -> str:
    h = socket.gethostname()
    try:
        socket.getaddrinfo(h, None)
        return h
    except OSError:
        return "127.0.0.1"


class _Server(ThreadingHTTPServer):
    address_family = socket.AF_INET6
    daemon_threads = True

    def server_bind(self) -> None:
        try:
            self.socket.setsockopt(socket.IPPROTO_IPV6, socket.IPV6_V6ONLY, 0)
        except OSError:
            pass
        super().server_bind()


class ParameterServer(ABC):
    """Prototype parameter server (reference: parameter_server.py:30-194): an HTTP endpoint hands out sessions, each session is a
    fresh 2-rank reconfigurable process group (server rank 0, client rank 1); subclasses implement ``new_process_group`` and ``forward``."""

    def __init__(self, port: int, store_port: int = 0) -> None:
        """
        Args:
            port: HTTP port for ``/new_session`` (0 = ephemeral)
            store_port: port of the TCPStore sessions rendezvous on (0 = ephemeral)
        """
        self.store = TCPStore(host_name="0.0.0.0", port=store_port, is_master=True, wait_for_workers=False)
        self._sessions: Dict[str, threading.Thread] = {}
        ps = self

        class Handler(BaseHTTPRequestHandler):
            def log_message(self, fmt: str, *args: object) -> None:
                logger.debug("parameter_server: " + fmt, *args)

            def do_GET(self) -> None:  # noqa: N802
                if self.path != "/new_session":
                    body = f"invalid path, got {self.path}".encode()
                    self.send_response(400)
                    self.send_header("Content-Type", "text/plain")
                    self.send_header("Content-Length", str(len(body)))
                    self.end_headers()
                    self.wfile.write(body)
                    return
                session_id = str(uuid.uuid4())
                store_addr = f"{_advertise_host()}:{ps.store.port}/session/{session_id}"
                body = (json.dumps({"session_id": session_id, "store_addr": store_addr}) + "\n").encode()
                self.send_response(200)
                self.send_header("Content-Type", "application/json")
                self.send_header("Content-Length", str(len(body)))
                self.end_headers()
                self.wfile.write(body)
                self.wfile.flush()
                t = threading.Thread(target=ps._handle_session, args=(session_id, store_addr),
                                     name=f"tft_ps_{session_id[:8]}", daemon=True)
                ps._sessions[session_id] = t
                t.start()

        self._server = _Server(("::", port), Handler)
        self._thread = threading.Thread(target=self._server.serve_forever, name="tft_ps_http", daemon=True)
        self._thread.start()
        logger.info("Started ParameterServer on %s", self.address())

    def address(self) -> str:
        """``http://host:port/new_session``"""
        return f"http://{_advertise_host()}:{self._server.socket.getsockname()[1]}/new_session"

    @classmethod
    @abstractmethod
    def new_process_group(cls) -> ProcessGroup:
        """A fresh, unconfigured process group (same class on server and client)."""

    @classmethod
    def new_session(cls, address: str) -> ProcessGroup:
        """Open a session; returns the client-side group (client = rank 1, server = rank 0)."""
        with urllib.request.urlopen(address) as f:
            data = json.load(f)
        logger.info("connecting to session %s at %s", data["session_id"], data["store_addr"])
        pg = cls.new_process_group()
        pg.configure(data["store_addr"], replica_id="0", rank=1, world_size=2)
        return pg

    def _handle_session(self, session_id: str, store_addr: str) -> None:
        try:
            pg = self.new_process_group()
            pg.configure(store_addr, replica_id="0", rank=0, world_size=2)
            self.forward(session_id, pg)
        except Exception:  # noqa: BLE001
            logger.exception("parameter server session %s failed", session_id)
        finally:
            self._sessions.pop(session_id, None)

    @abstractmethod
    def forward(self, session_id: str, pg: ProcessGroup) -> None:
        """Serve one session (loop inside for multiple operations). Server rank 0, client rank 1.
        On error the group is dropped and the client must open a new session."""

    def shutdown(self) -> None:
        self._server.shutdown()
        self._server.server_close()
