"""The MatcherParser stage on the H100 (B200MatcherParser, dm_parse_logs; rule R-parse in DESIGN.md).

- Byte identity: the device path returns the host path's bytes on the generators of test_matcher_parser.py, on 64k-
  record batches of both log formats, on one 8 MiB record and across the growth of the output buffer.
- Split = fused: B200MatcherParser -> B200NewValueDetector(parser_schema_batch) flags and scores every emitted record as
  B200NewValueDetector(log_schema_batch) with the same log_format does, and with a fixed clock replies the same bytes.
- Three services: reader -> the unmodified reference Service with B200MatcherParser and the reference's
  parser_config.yaml -> the same Service with B200NewValueDetector and the reference's detector_config.yaml -> sink.
"""
import os
import random
import time

import numpy as np
import pytest
import yaml

from detectmateservice_b200 import wire
from detectmateservice_b200.component import B200NewValueComboDetector, B200NewValueDetector, decode_compact
from test_matcher_parser import (CASES, GOLDEN, NGINX, NOW, audit_case, decoded, log_records, make_case,
                                 nginx_line, oracle_fields, parser)

pytestmark = pytest.mark.gpu


def _same(comp_dev, comp_host, msg, delimited=True):
    dev = comp_dev._parse_device(msg, delimited)
    host = comp_host._parse_host(msg, delimited)
    assert dev == host
    assert comp_dev.n_parsed == comp_host.n_parsed and comp_dev.last_n_malformed == comp_host.last_n_malformed
    return dev


@pytest.mark.parametrize("kind,seed,norm", CASES)
def test_device_matches_host(kind, seed, norm):
    comp_host, recs = make_case(kind, seed, norm, n_records=3000)
    comp_dev, _ = make_case(kind, seed, norm, n_records=3000)
    try:
        half = len(recs) // 3
        for part in (recs[:half], recs[half:]):
            _same(comp_dev, comp_host, wire.frame_delimited(part))
        for rec in recs[:40]:                                    # bare records, on the device too
            try:
                host = comp_host._parse_host(rec, False)
            except wire.WireError:
                with pytest.raises(wire.WireError):
                    comp_dev._parse_device(rec, False)
                continue
            assert comp_dev._parse_device(rec, False) == host
        assert comp_dev._parse_device(b"", True) is None
    finally:
        comp_dev.close()


def _nginx_64k(seed):
    r = random.Random(seed)
    lines = [nginx_line("/p%d" % r.randrange(5000), "10.%d.%d.%d" % (r.randrange(9), r.randrange(256), r.randrange(256)))
             for _ in range(65536)]
    return parser(NGINX), lines


def test_64k_batches_both_formats_and_growth():
    """64k-record batches of the nginx and the audit format (+ templates, all three R-norm switches); a small batch
    first, so that the big ones outgrow the output buffer the first call allocated."""
    audit_lines = [ln for ln in open(os.path.join(GOLDEN, "audit_sample.log"), "rb").read().split(b"\n") if ln]
    for make in ("nginx", "audit"):
        if make == "nginx":
            comp_dev, lines = _nginx_64k(1)
            comp_host, _ = _nginx_64k(1)
        else:
            comp_dev, _r = audit_case(2)
            comp_host, _r = audit_case(2)
            lines = [audit_lines[i % len(audit_lines)] for i in range(65536)]
        try:
            recs = log_records(lines, 3, mutate=0.01)
            _same(comp_dev, comp_host, wire.frame_delimited(recs[:10]))
            out = _same(comp_dev, comp_host, wire.frame_delimited(recs))
            assert len(out) > 4 << 20                            # (the first call's buffer held 1 MiB)
            want = [d for d in oracle_fields(comp_dev, recs[:500], 10) if d is not None]
            assert decoded(out)[:len(want)] == want
        finally:
            comp_dev.close()


def test_one_8mib_record():
    comp_dev, comp_host = parser(NGINX), parser(NGINX)
    try:
        big = nginx_line("/" + "a" * (8 << 20))
        rec = wire.encode_log_schema({"logID": "big", "log": big.decode() + "\n"})
        out = _same(comp_dev, comp_host, wire.frame_delimited([rec, rec[:100]]))
        assert decoded(out)[0]["logFormatVariables"]["URL"] == "/" + "a" * (8 << 20)
        assert comp_dev._parse_device(rec, False) == comp_host._parse_host(rec, False)
    finally:
        comp_dev.close()


# ------------------------------------------------------------------------------------------ split = fused
def _detector(cls, training, input_format, log_format=None, combo=False):
    glob = {"g": {"header_variables": [{"pos": "URL"}, {"pos": "Status"}]}} if combo else \
        {"g": {"header_variables": [{"pos": "URL"}]}, "h": {"header_variables": [{"pos": "IP"}]}}
    params = {"input_format": input_format}
    if log_format:
        params["log_format"] = log_format
    name = "NewValueComboDetector" if combo else "NewValueDetector"
    det = cls(config={"detectors": {name: {"method_type": "x", "data_use_training": training, "global": glob,
                                           "params": params}}})
    det.clock = lambda: NOW
    return det


@pytest.mark.parametrize("combo", [False, True])
def test_split_equals_fused(combo):
    cls = B200NewValueComboDetector if combo else B200NewValueDetector
    r = random.Random(7)
    lines = [nginx_line("/p%d" % r.randrange(60 if i < 3000 else 80), "10.0.0.%d" % r.randrange(30 if i < 3000 else 40))
             for i in range(6000)]
    lines[100] = b"not an access-log line"                       # a rejected line keeps its training slot
    recs = log_records(lines, 8, mutate=0.02)
    msgs = [wire.frame_delimited(recs[:2500]), wire.frame_delimited(recs[2500:])]   # training ends inside the first
    for output in ("compact", "alerts"):
        p = parser(NGINX)
        fused = _detector(cls, 2000, "log_schema_batch", NGINX, combo)
        split = _detector(cls, 2000, "parser_schema_batch", combo=combo)
        fused.output_format = split.output_format = output
        flagged = 0
        try:
            for m in msgs:
                a = fused.process(m)
                b = split.process(p.process(m))
                if output == "alerts":
                    assert a == b
                    flagged += len(wire.split_delimited(b or b""))
                    continue
                fa, sa = decode_compact(a)
                fb, sb = decode_compact(b)
                usable = [i for i, rec in enumerate(wire.split_delimited(m)) if _usable(rec)]
                assert np.array_equal(fa[usable], fb) and np.array_equal(sa[usable], sb)
                flagged += int(fb.sum())
            assert flagged > 0
        finally:
            p.close()
            fused.close()
            split.close()


def _usable(rec):
    try:
        wire.log_schema_line(wire.decode_log_schema(rec))
        return True
    except wire.WireError:
        return False


# ------------------------------------------------------------------------------------------ three services
def _reference_src():
    from oracle.ref_engine import reference_path
    return reference_path()


@pytest.mark.skipif(_reference_src() is None, reason="the reference service is not in oracle/_ref (make -C oracle ref)")
def test_reference_services_reader_parser_detector(tmp_path, ipc_dir, monkeypatch):
    """reader -> B200MatcherParser -> B200NewValueDetector, each stage the unmodified reference Service; the docs'
    /hello, /world, /foobar give the alert of docs/getting_started.md on /foobar."""
    from detectmateservice_b200.compat import install_shims
    monkeypatch.syspath_prepend(_reference_src())
    install_shims()
    import pynng
    from service.core import Service
    from service.settings import ServiceSettings

    pcfg = yaml.safe_load(open(os.path.join(GOLDEN, "parser_config.yaml")))
    (tmp_path / "templates.txt").write_bytes(b"")
    pcfg["parsers"]["MatcherParser"]["params"]["path_templates"] = str(tmp_path / "templates.txt")
    (tmp_path / "parser_config.yaml").write_text(yaml.safe_dump(pcfg))
    a_parser, a_det, a_sink = (f"ipc://{ipc_dir}/{n}.ipc" for n in ("parser", "detector", "sink"))
    with pynng.Pair0(listen=a_sink, recv_timeout=5000) as sink:
        services = []
        try:
            for name, cls, cfg, addr, out in (
                    ("b200-detector", "detectmateservice_b200.component.B200NewValueDetector",
                     os.path.join(GOLDEN, "detector_config.yaml"), a_det, a_sink),
                    ("b200-parser", "detectmateservice_b200.parser.B200MatcherParser", tmp_path / "parser_config.yaml",
                     a_parser, a_det)):
                s = Service(settings=ServiceSettings(
                    component_type=cls, component_name=name, engine_addr=addr, out_addr=[out], config_file=cfg,
                    log_dir=tmp_path / "logs", log_to_file=False, log_to_console=False,
                    http_port=18240 + len(services), engine_autostart=False))
                s.start()
                services.append(s)
            time.sleep(0.3)
            with pynng.Pair0(dial=a_parser) as reader:
                time.sleep(0.2)
                for i, url in enumerate(("/hello", "/world", "/foobar")):
                    rec = wire.encode_log_schema({"__version__": "1.0.0", "logID": "reader-%d" % i,
                                                  "log": nginx_line(url).decode() + "\n"})
                    reader.send(wire.frame_delimited([rec]))
                alerts = [wire.decode_detector_schema(m) for m in wire.split_delimited(sink.recv())]
            assert len(alerts) == 1
            assert alerts[0]["alertsObtain"] == {"Global - URL": "Unknown value: '/foobar'"}
            assert alerts[0]["logIDs"] == ["reader-2"] and alerts[0]["detectorID"] == "NewValueDetector"
        finally:
            for s in services:
                s.stop()
            for s in services:
                s.library_component.close()
