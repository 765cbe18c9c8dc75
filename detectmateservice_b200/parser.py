"""B200MatcherParser -- the reference pipeline's parser stage (reader -> parser -> detector) on libdmdetect.

Stands where ``detectmatelibrary.parsers.template_matcher.MatcherParser`` stands behind the UNMODIFIED reference
service (container/config/parser_settings.yaml, docs/getting_started.md "Parser"): LogSchema records in, one
ParserSchema per record out, so that several detectors -- the library's, a user's CustomDetector, or
B200NewValueDetector with ``input_format: parser_schema_batch`` -- can sit behind one parser.

  settings YAML   component_type: detectmateservice_b200.parser.B200MatcherParser
  config YAML     the reference's own parser config (container/config/parser_config.yaml): ``parsers: {<name>:
                  {method_type, auto_config, log_format, time_format, params: {remove_spaces, remove_punctuation,
                  lowercase, path_templates}}}``, the entry named as the component or ``MatcherParser``.  Further
                  ``params``: templates (a list, before those of path_templates), content_name ("Content"), parser_id
                  ("MatcherParser" when the component's name starts with B200, else the name), start_id (0),
                  input_format (log_schema | log_schema_batch, default log_schema_batch), device, max_batch_bytes.

Rule R-parse (DESIGN.md) says what a record becomes; the host path here (_parse_host) is its specification.  A
varint-length-delimited batch is parsed on the device (dm_parse_logs), byte for byte what the host path writes; a
bare record is parsed on the host, because one record does not pay for the device's launches and two synchronisations
(scripts/parser_bench.py measures both sides).  A malformed bare record raises WireError; in a batch it gives no
output.  Replies: a bare ParserSchema for a bare record, the varint-delimited ParserSchemas of a batch, None when a
batch emits nothing.
"""
from __future__ import annotations

import threading
import time
from typing import Any, Optional, Tuple

from . import wire
from .component import B200NewValueDetector, select_component_config
from .compat import install_shims
from .logformat import LogFormat, load_templates, norm_flags

install_shims()
from detectmatelibrary.common.core import CoreComponent, CoreConfig  # noqa: E402

PARSER_INPUT_FORMATS = ("log_schema", "log_schema_batch")


class B200MatcherParserConfig(CoreConfig):
    """Schema of the parser's config entry (found by the resolver as <Class>Config in the same module)."""
    method_type: str = "matcher_parser"
    auto_config: bool = False


class B200MatcherParser(CoreComponent):
    accepts_bytes_like = True      # process() takes bytes, bytearray or memoryview (see service.py)

    def __init__(self, name: str = "B200MatcherParser", config: Optional[Any] = None) -> None:
        raw_cfg = config.model_dump() if hasattr(config, "model_dump") else config
        cfg = select_component_config(raw_cfg, name, fallback="MatcherParser", section="parsers")
        self.method_type = str(cfg.get("method_type", "matcher_parser"))
        super().__init__(name=name, config=B200MatcherParserConfig(method_type=self.method_type,
                                                                   auto_config=bool(cfg.get("auto_config", False))))
        if cfg.get("auto_config"):
            raise ValueError("auto_config: true (a configure phase) is not supported by the CUDA parser; give log_format "
                             "and the templates")
        if cfg.get("time_format") is not None:
            raise ValueError("time_format: only null is supported (Time is passed on as the text it is)")
        if not cfg.get("log_format"):
            raise ValueError("log_format is missing: the CUDA parser splits records by a log_format")
        templates = list(cfg.get("templates") or [])
        if cfg.get("path_templates"):
            templates += load_templates(str(cfg["path_templates"]))
        templates = [t if isinstance(t, bytes) else str(t).encode("utf-8") for t in templates]
        for i, t in enumerate(templates):
            try:
                t.decode("utf-8")
            except UnicodeDecodeError:
                raise ValueError(f"template {i} is not valid UTF-8") from None
        flags = norm_flags(bool(cfg.get("remove_spaces")), bool(cfg.get("remove_punctuation")), bool(cfg.get("lowercase")))
        self.logformat = LogFormat(cfg["log_format"], templates, str(cfg.get("content_name", "Content")), flags)
        self.parser_id = str(cfg.get("parser_id", "MatcherParser" if name.startswith("B200") else name))
        self.start_id = int(cfg.get("start_id", 0))
        self.input_format = cfg.get("input_format", "log_schema_batch")
        if self.input_format not in PARSER_INPUT_FORMATS:
            raise ValueError(f"input_format {self.input_format!r} not in {'|'.join(PARSER_INPUT_FORMATS)}")
        self.device = int(cfg.get("device", 0))
        self.max_batch_bytes = int(cfg.get("max_batch_bytes", 64 << 20))
        self._det = None                       # created on first use, on the EngineLoop thread
        self._frames = None                    # pinned receive slots, created on first alloc_frame()
        self._frame_lock = threading.Condition()
        self.n_parsed = 0                      # ParserSchemas emitted: the next parsedLogID is start_id + n_parsed
        self.last_n_malformed = 0
        self.clock = time.time

    # ------------------------------------------------------------------ device handle
    @property
    def det(self):
        if self._det is None:
            from .detector import DeviceDetector
            lf = self.logformat
            d = DeviceDetector([], device=self.device, max_batch_bytes=self.max_batch_bytes, table_log2_slots=10)
            d.set_monitors([])
            d.set_format(lf.source, lf.template_sources, lf.content_name, lf.flags)
            d.set_parser_format("1.0.0", self.method_type, self.parser_id, lf.template_sources, lf.header.names)
            self._det = d
        return self._det

    # receive buffers lent to the transport: pinned slots, as the detector lends them
    FRAME_SLOTS = B200NewValueDetector.FRAME_SLOTS
    alloc_frame = B200NewValueDetector.alloc_frame
    release_frame = B200NewValueDetector.release_frame

    def close(self) -> None:
        if self._det is not None:
            self._det.close()
            self._det = None

    # ------------------------------------------------------------------ the plugin entry point
    def process(self, data: bytes) -> Optional[bytes]:
        delimited = self.input_format == "log_schema_batch"
        if delimited and not data:
            return None
        if len(data) > self.max_batch_bytes:
            raise ValueError(f"a LogSchema message of {len(data)} bytes exceeds max_batch_bytes={self.max_batch_bytes}")
        if delimited:
            return self._parse_device(data, delimited=True)
        return self._parse_host(bytes(data), delimited=False)

    def _parse_device(self, data, delimited: bool) -> Optional[bytes]:
        """R-parse on the device (dm_parse_logs)."""
        now = int(self.clock())
        out, _n, n_emitted, n_bad = self.det.parse_logs(data, delimited, self.start_id + self.n_parsed, now)
        self.last_n_malformed = n_bad
        if not delimited and n_bad:
            raise wire.WireError("malformed LogSchema record")
        self.n_parsed += n_emitted
        if delimited:
            return out or None
        _ln, pos = wire._read_varint(out, 0)                    # one record in, one bare ParserSchema out
        return out[pos:]

    def _parse_host(self, data: bytes, delimited: bool) -> Optional[bytes]:
        """R-parse on the host, one record at a time: the specification the device path is held to."""
        now = int(self.clock())
        frames = wire.split_delimited(data) if delimited else [data]
        out, bad = [], 0
        for fr in frames:
            try:
                rec = wire.decode_log_schema(fr)
                text = wire.log_schema_line(rec)
            except wire.WireError:
                if not delimited:
                    raise
                bad += 1
                continue
            out.append(self._parser_schema(rec["logID"], text, now))
        self.last_n_malformed = bad
        if not delimited:
            return out[0]
        return wire.frame_delimited(out) if out else None

    def _parser_schema(self, log_id: str, text: bytes, now: int) -> bytes:
        """The ParserSchema of one usable record (R-parse 2-3)."""
        rec = {"__version__": "1.0.0", "parserType": self.method_type, "parserID": self.parser_id}
        parsed: Optional[Tuple] = self.logformat.parse(text)
        if parsed is None:
            rec["EventID"] = -1
        else:
            eid, variables, lfv = parsed
            rec["EventID"] = eid
            if eid >= 0:
                rec["template"] = self.logformat.template_sources[eid]
            rec["variables"] = variables
            rec["logFormatVariables"] = lfv
        rec["parsedLogID"] = str(self.start_id + self.n_parsed)
        self.n_parsed += 1
        rec["logID"] = log_id
        rec["log"] = text
        rec["receivedTimestamp"] = rec["parsedTimestamp"] = now
        return wire.encode_parser_schema(rec)
