"""Engine loop mirror + service wrappers for the CUDA detector.

Two ways to run the detector behind the reference's data channel:

1. Inside the UNMODIFIED reference service (preferred when it is installed): point the
   settings YAML at ``detectmateservice_b200.component.B200NewValueDetector`` -- nothing in
   this module is needed -- or subclass the reference's ``Service`` (``b200_detector_service()``
   below; the subclass route of /root/reference/src/service/core.py:64-69,85-86 that every
   in-process reference test uses, tests/test_engine_loop.py:12-20).

2. Stand-alone (no reference checkout, e.g. on a bare GPU box): ``DetectorEngine`` is a
   from-scratch mirror of the reference's hot loop ``Engine._run_loop``
   (/root/reference/src/service/features/engine.py:153-217) with the same observable
   behaviour: one PAIR0 listener on ``engine_addr``; every non-empty message goes through
   ``processor.process``; ``None`` => nothing is sent; an exception => logged, message
   dropped, loop continues; a result is sent non-blocking to every ``out_addr`` (dropped and
   counted on ``TryAgain``, engine.py:219-244) or, with no outputs configured, replied on the
   input socket (engine.py:204-217).  ``stop()`` joins the loop within 2 s (engine.py:262-265).
"""
from __future__ import annotations

import logging
import threading
from typing import Any, Dict, List, Optional, Sequence

from .compat import install_shims

install_shims()
import pynng  # noqa: E402  (the real package, or the SP/PAIR0 shim)


class DetectorEngine:
    def __init__(self, processor: Any, engine_addr: str, out_addr: Sequence[str] = (), recv_timeout_ms: int = 100,
                 out_dial_timeout_ms: int = 1000, logger: Optional[logging.Logger] = None) -> None:
        if processor is None or not hasattr(processor, "process"):
            raise ValueError("DetectorEngine requires a processor with a process() method")
        self.processor = processor
        self.log = logger or logging.getLogger("detectmateservice_b200.engine")
        self.counters: Dict[str, int] = {"read_bytes": 0, "written_bytes": 0, "dropped_bytes": 0,
                                         "processed_lines": 0, "messages": 0, "errors": 0}
        self._running = False
        self._stop = threading.Event()
        self._thread: Optional[threading.Thread] = None
        self._sock = pynng.Pair0()
        self._sock.recv_timeout = recv_timeout_ms
        try:
            self._sock.recv_max_size = 0           # batches are multi-MiB messages: no receive limit (NNG's default is 1 MiB)
        except Exception:                          # (a pynng build without the option: keep its default)
            pass
        # shim-only hint (ignored by real pynng): hand big frames over as a bytearray filled in
        # place; the component takes any bytes-like object, and this halves the receive cost
        self._sock.large_frames_as_bytearray = bool(getattr(processor, "accepts_bytes_like", False))
        # a processor may lend receive buffers (alloc_frame / release_frame): the component hands
        # out pinned host memory, so a frame lands where the GPU can DMA it from (no extra copy)
        self._release = getattr(processor, "release_frame", None)
        if self._release is not None and hasattr(processor, "alloc_frame"):
            self._sock.frame_allocator = processor.alloc_frame
        self._sock.listen(engine_addr)
        self._outs: List[Any] = []
        for addr in out_addr:
            s = pynng.Pair0()
            s.dial_timeout = out_dial_timeout_ms
            s.send_buffer_size = 0
            s.recv_buffer_size = 0
            s.dial(str(addr), block=False)          # background connect, late binding
            self._outs.append(s)

    def start(self) -> str:
        if self._running:
            return "engine already running"
        self._running = True
        self._stop.clear()
        self._thread = threading.Thread(target=self._run_loop, name="EngineLoop", daemon=True)
        self._thread.start()
        return "engine started"

    def _run_loop(self) -> None:
        c = self.counters
        while self._running and not self._stop.is_set():
            try:
                raw = self._sock.recv()
            except pynng.Timeout:
                continue
            except pynng.NNGException as e:
                if not self._running or self._stop.is_set():
                    break
                self.log.error("engine error during receive: %s", e)
                continue
            if not raw:
                continue
            c["read_bytes"] += len(raw)
            c["messages"] += 1
            # core.py:190 counts '\n' on the host (15 ms for a 16 MiB message); a processor that
            # already counts records (the component's n_seen, taken from the GPU's line index)
            # supplies the same number for free
            seen0 = getattr(self.processor, "n_seen", None)
            if seen0 is None:
                c["processed_lines"] += raw.count(b"\n") or 1
            try:
                out = self.processor.process(raw)
                if seen0 is not None:
                    c["processed_lines"] += (self.processor.n_seen - seen0) or 1
            except Exception as e:                               # engine.py:192-194
                c["errors"] += 1
                self.log.exception("engine error during process: %s", e)
                continue
            finally:
                if self._release is not None:
                    self._release(raw)                           # the frame buffer may be reused now
            if out is None:
                continue
            if self._outs:
                for i, s in enumerate(self._outs):
                    try:
                        s.send(out, block=False)
                        c["written_bytes"] += len(out)
                    except pynng.TryAgain:
                        c["dropped_bytes"] += len(out)
                    except pynng.NNGException as e:
                        self.log.error("engine error sending to output %d: %s", i, e)
            else:
                try:
                    self._sock.send(out)
                    c["written_bytes"] += len(out)
                except pynng.NNGException as e:
                    self.log.error("engine error sending reply: %s", e)

    def stop(self) -> None:
        if not self._running:
            return
        self._running = False
        self._stop.set()
        if self._thread is not None:
            self._thread.join(timeout=2.0)
            if self._thread.is_alive():
                raise RuntimeError("engine thread failed to stop cleanly")
        self._sock.close()
        for s in self._outs:
            try:
                s.close()
            except pynng.NNGException:
                pass

    def __enter__(self):
        self.start()
        return self

    def __exit__(self, *exc):
        self.stop()
        return False


def b200_detector_service():
    """Return a ``Service`` subclass bound to the CUDA detector (needs the reference's
    ``service`` package importable).  Usage::

        B200DetectorService = b200_detector_service()
        svc = B200DetectorService(settings=ServiceSettings(...), component_config={...})
        with svc: svc.run()
    """
    from service.core import Service  # the reference package
    from .component import B200NewValueDetector

    class B200DetectorService(Service):
        component_type = "detectmateservice_b200.component.B200NewValueDetector"

        def __init__(self, settings=None, component_config: Optional[dict] = None):
            from service.settings import ServiceSettings
            super().__init__(settings=settings if settings is not None else ServiceSettings(),
                             component_config=component_config)
            cfg = component_config
            if cfg is None and self.config_manager is not None:
                got = self.config_manager.get()
                cfg = got.model_dump() if hasattr(got, "model_dump") else got
            self.detector = B200NewValueDetector(config=cfg or {})

        def process(self, raw_message: bytes):
            # keep the base class's metrics (core.py:184-200) by routing through it
            self.library_component = self.detector
            if self._pending_config is not None:             # (applied on the engine thread, between two messages)
                cfg, self._pending_config = self._pending_config, None
                self.detector.reconfigure(cfg)
            return super().process(raw_message)

        _pending_config = None

        def reconfigure(self, config_data, persist: bool = False) -> str:
            # the reference validates + stores the new configuration (core.py:299-345); the detector takes it over
            # before the next message
            out = super().reconfigure(config_data, persist=persist)
            if out == "reconfigure: ok" and self.config_manager is not None:
                got = self.config_manager.get()
                self._pending_config = got.model_dump() if hasattr(got, "model_dump") else got
            return out

    return B200DetectorService
