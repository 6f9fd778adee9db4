"""Structured-event export for the ``torchft_quorums`` / ``torchft_commits`` /
``torchft_errors`` loggers.

Two sinks, both opt-in through the environment:

* ``TORCHFT_USE_OTEL=true`` -- ship records through OpenTelemetry (OTLP + console),
  with per-logger resource attributes from the JSON file named by
  ``TORCHFT_OTEL_RESOURCE_ATTRIBUTES_JSON`` (same switches as the reference,
  upstream torchft/otel.py:44-103). Needs the ``opentelemetry`` SDK; a clear
  error is raised if it is requested but missing.
* ``TORCHFT_B200_EVENTS_JSONL=/path/file.jsonl`` -- dependency-free JSON-lines sink
  (one object per quorum / commit / error event with job_id, replica_id, rank,
  quorum_id, step, ...), handy on air-gapped clusters and in tests.
* ``TORCHFT_B200_PROMETHEUS_PORT=9400`` -- a Prometheus scrape endpoint fed by the same three loggers
  (ours; needs ``prometheus_client``): ``torchft_quorum_changes_total``, ``torchft_commits_total{result=}``,
  ``torchft_errors_total``, ``torchft_step``, ``torchft_quorum_id``, all labelled with ``replica_id`` / ``rank``.
"""

from __future__ import annotations

import json
import logging
import os
import threading
import time
from typing import Any, Dict

TORCHFT_OTEL_RESOURCE_ATTRIBUTES_JSON = "TORCHFT_OTEL_RESOURCE_ATTRIBUTES_JSON"
TORCHFT_USE_OTEL = "TORCHFT_USE_OTEL"
EVENTS_JSONL_ENV = "TORCHFT_B200_EVENTS_JSONL"
PROMETHEUS_PORT_ENV = "TORCHFT_B200_PROMETHEUS_PORT"

_PROVIDERS: Dict[str, Any] = {}
_JSONL: Dict[str, logging.Handler] = {}
_STD_ATTRS = set(logging.LogRecord("", 0, "", 0, "", (), None).__dict__) | {"message", "asctime"}


class JsonLinesHandler(logging.Handler):
    """Append each record's structured ``extra`` fields as one JSON object per line."""

    def __init__(self, path: str, logger_name: str) -> None:
        super().__init__(level=logging.NOTSET)
        self._path, self._name = path, logger_name
        self._lock = threading.Lock()

    def emit(self, record: logging.LogRecord) -> None:
        try:
            event = {"logger": self._name, "ts": time.time(), "level": record.levelname, "msg": record.getMessage()}
            for k, v in record.__dict__.items():
                if k not in _STD_ATTRS and not k.startswith("_"):
                    try:
                        json.dumps(v)
                        event[k] = v
                    except TypeError:
                        event[k] = repr(v)
            with self._lock, open(self._path, "a") as f:
                f.write(json.dumps(event) + "\n")
        except Exception:  # pragma: no cover
            self.handleError(record)


class PrometheusHandler(logging.Handler):
    """Turns quorum / commit / error records into Prometheus counters and gauges (one registry per process)."""

    _lock = threading.Lock()
    _metrics: Dict[str, Any] = {}
    _server_port: Any = None

    @classmethod
    def _ensure(cls, port: int) -> Dict[str, Any]:
        with cls._lock:
            if not cls._metrics:
                try:
                    import prometheus_client as pc
                except ImportError as e:
                    raise RuntimeError(f"{PROMETHEUS_PORT_ENV} is set but prometheus_client is not installed: {e}") from e
                labels = ["replica_id", "rank"]
                cls._metrics = {
                    "quorums": pc.Counter("torchft_quorum_changes_total", "quorum reconfigurations seen by this rank", labels),
                    "commits": pc.Counter("torchft_commits_total", "should_commit verdicts", labels + ["result"]),
                    "errors": pc.Counter("torchft_errors_total", "process-group errors / aborts", labels),
                    "step": pc.Gauge("torchft_step", "last step seen in a quorum or commit event", labels),
                    "quorum_id": pc.Gauge("torchft_quorum_id", "current quorum id", labels),
                }
                if port > 0:
                    pc.start_http_server(port)
                    cls._server_port = port
            return cls._metrics

    def __init__(self, logger_name: str, port: int) -> None:
        super().__init__(level=logging.NOTSET)
        self._name = logger_name
        self._m = self._ensure(port)

    def emit(self, record: logging.LogRecord) -> None:
        try:
            d = record.__dict__
            lab = {"replica_id": str(d.get("replica_id", "")), "rank": str(d.get("rank", ""))}
            if self._name == "torchft_quorums":
                self._m["quorums"].labels(**lab).inc()
            elif self._name == "torchft_commits":
                self._m["commits"].labels(result="committed" if d.get("commit_result") else "failed", **lab).inc()
            elif self._name == "torchft_errors":
                self._m["errors"].labels(**lab).inc()
            if isinstance(d.get("step"), int):
                self._m["step"].labels(**lab).set(d["step"])
            if isinstance(d.get("quorum_id"), int):
                self._m["quorum_id"].labels(**lab).set(d["quorum_id"])
        except Exception:  # pragma: no cover
            self.handleError(record)


_PROM: Dict[str, logging.Handler] = {}


def _setup_otel(name: str) -> None:
    try:
        from opentelemetry._logs import set_logger_provider
        from opentelemetry.exporter.otlp.proto.http._log_exporter import OTLPLogExporter
        from opentelemetry.sdk._logs import LoggerProvider, LoggingHandler
        from opentelemetry.sdk._logs.export import BatchLogRecordProcessor, ConsoleLogExporter
        from opentelemetry.sdk.resources import Resource
    except ImportError as e:
        raise RuntimeError(f"{TORCHFT_USE_OTEL}=true but the opentelemetry SDK is not installed: {e}") from e
    attrs_file = os.environ.get(TORCHFT_OTEL_RESOURCE_ATTRIBUTES_JSON)
    if attrs_file is not None:
        with open(attrs_file) as f:
            resource = Resource.create(attributes=json.load(f)[name])
    else:
        resource = Resource.create()
    provider = LoggerProvider(resource=resource)
    set_logger_provider(provider)
    for exporter in (ConsoleLogExporter(), OTLPLogExporter(timeout=5)):
        provider.add_log_record_processor(BatchLogRecordProcessor(exporter))
    logging.getLogger(name).addHandler(LoggingHandler(level=logging.NOTSET, logger_provider=provider))
    _PROVIDERS[name] = provider


def setup_logger(name: str) -> None:
    """Attach the configured sinks to logger ``name`` (idempotent)."""

    logger = logging.getLogger(name)
    path = os.environ.get(EVENTS_JSONL_ENV)
    if path and name not in _JSONL:
        h = JsonLinesHandler(path, name)
        logger.addHandler(h)
        if logger.level == logging.NOTSET or logger.level > logging.INFO:
            logger.setLevel(logging.INFO)
        _JSONL[name] = h
    port = os.environ.get(PROMETHEUS_PORT_ENV)
    if port and name not in _PROM:
        h = PrometheusHandler(name, int(port))
        logger.addHandler(h)
        if logger.level == logging.NOTSET or logger.level > logging.INFO:
            logger.setLevel(logging.INFO)
        _PROM[name] = h
    if os.environ.get(TORCHFT_USE_OTEL, "false") != "false" and name not in _PROVIDERS:
        _setup_otel(name)


def shutdown() -> None:
    for p in _PROVIDERS.values():
        p.shutdown()
    _PROVIDERS.clear()
    for name, h in _JSONL.items():
        logging.getLogger(name).removeHandler(h)
    _JSONL.clear()
    for name, h in _PROM.items():
        logging.getLogger(name).removeHandler(h)
    _PROM.clear()
