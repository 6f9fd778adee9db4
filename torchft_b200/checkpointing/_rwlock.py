"""Timed readers-writer lock built on one condition variable.

Parity with the reference's ``RWLock``
(upstream torchft/checkpointing/_rwlock.py:46-136): every acquire takes
at most ``timeout`` seconds and raises ``TimeoutError`` otherwise. Unlike the
two-mutex construction used there, the write side here may be released from a
different thread than the one that acquired it (the Manager takes it on the
training thread and a transport may release it from its server thread) and
waiting writers block new readers, so a steady stream of checkpoint fetches
cannot starve ``disallow_checkpoint``.
"""

from __future__ import annotations

import threading
import time
from contextlib import contextmanager
from typing import Generator


class RWLock:
    """Reader-writer lock with timeouts (reference: checkpointing/_rwlock.py:46-136): many readers or one writer;
    ``r_lock()`` / ``w_lock()`` are context managers, acquisition raises ``TimeoutError`` after ``timeout`` seconds."""

    def __init__(self, timeout: float = -1) -> None:
        self.timeout = timeout
        self._cv = threading.Condition(threading.Lock())
        self._readers = 0
        self._writer = False
        self._writers_waiting = 0

    def _deadline(self) -> float | None:
        return None if self.timeout is None or self.timeout < 0 else time.monotonic() + self.timeout

    def _wait(self, deadline: float | None, what: str) -> None:
        if deadline is None:
            self._cv.wait()
            return
        remaining = deadline - time.monotonic()
        if remaining <= 0 or not self._cv.wait(remaining):
            if deadline - time.monotonic() <= 0:
                raise TimeoutError(f"Timed out waiting for {what} after {self.timeout} seconds")

    # ---- readers ----
    def r_acquire(self) -> None:
        deadline = self._deadline()
        with self._cv:
            while self._writer or self._writers_waiting:
                self._wait(deadline, "rlock")
            self._readers += 1

    def r_release(self) -> None:
        with self._cv:
            assert self._readers > 0, "r_release without r_acquire"
            self._readers -= 1
            if self._readers == 0:
                self._cv.notify_all()

    @contextmanager
    def r_lock(self) -> Generator[None, None, None]:
        self.r_acquire()
        try:
            yield
        finally:
            self.r_release()

    # ---- writer ----
    def w_acquire(self) -> None:
        deadline = self._deadline()
        with self._cv:
            self._writers_waiting += 1
            try:
                while self._writer or self._readers:
                    self._wait(deadline, "wlock")
                self._writer = True
            finally:
                self._writers_waiting -= 1
                if not self._writer:
                    self._cv.notify_all()

    def w_release(self) -> None:
        with self._cv:
            assert self._writer, "w_release without w_acquire"
            self._writer = False
            self._cv.notify_all()

    @contextmanager
    def w_lock(self) -> Generator[None, None, None]:
        self.w_acquire()
        try:
            yield
        finally:
            self.w_release()

    def w_locked(self) -> bool:
        """True while a writer holds the lock or readers hold it exclusively of writers."""
        with self._cv:
            return self._writer or self._readers > 0
