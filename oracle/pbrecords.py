"""Record-mode oracle: length-delimited ParserSchema records judged by protobuf's own runtime.  TEST INFRASTRUCTURE.

Each frame is parsed with upb (``oracle.schemas.ParserSchema.ParseFromString``), the runtime the reference's
Python stack uses.  A frame upb refuses is malformed; so is a frame holding a group (wire types 3/4), the one
deliberate divergence of the product from upb (DESIGN.md section 5.3): upb keeps a group as an unknown field, and a
map entry that carried one among its unknown fields, so both are found there.  Every accepted record becomes the
oracle's dict (values as str; the detector oracles hash them as UTF-8 bytes) and steps NewValueDetectorOracle, or
NewValueComboDetectorOracle, in order: training is counted by rank among the well-formed records.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import List, Optional

from google.protobuf import message, message_factory
from google.protobuf.unknown_fields import UnknownFieldSet

from .nvcd import NewValueComboDetectorOracle
from .nvd import NewValueDetectorOracle
from .schemas import ParserSchema

_ENTRY = message_factory.GetMessageClass(ParserSchema.DESCRIPTOR.fields_by_name["logFormatVariables"].message_type)
_WT_GROUP = 3


def _has_group(msg) -> bool:
    for f in UnknownFieldSet(msg):
        if f.wire_type == _WT_GROUP:
            return True
        if f.field_number == 10 and f.wire_type == 2:            # a map entry upb dropped for its unknown fields
            e = _ENTRY()
            e.ParseFromString(f.data)
            if _has_group(e):
                return True
    return False


def parse(frame: bytes) -> Optional[dict]:
    """The oracle's record dict, or None if the frame is malformed."""
    m = ParserSchema()
    try:
        m.ParseFromString(frame)
    except message.DecodeError:
        return None
    if _has_group(m):
        return None
    return {"EventID": m.EventID if m.HasField("EventID") else None, "variables": list(m.variables),
            "logFormatVariables": dict(m.logFormatVariables), "logID": m.logID}


@dataclass
class Run:
    oracle: NewValueDetectorOracle
    flags: List[int] = field(default_factory=list)
    scores: List[float] = field(default_factory=list)
    masks: List[int] = field(default_factory=list)
    ok: List[bool] = field(default_factory=list)
    outputs: List[bytes] = field(default_factory=list)   # serialized DetectorSchema of every flagged record, in order

    @property
    def n_bad(self) -> int:
        return self.ok.count(False)

    def feed(self, frames: List[bytes]) -> "Run":
        """Steps the oracle through `frames`; appends one (flag, score, mask) per frame (0, 0, 0 if malformed)."""
        orc = self.oracle
        combos = getattr(orc, "combos", None)
        for fr in frames:
            rec = parse(fr)
            self.ok.append(rec is not None)
            if rec is None:
                self.flags.append(0); self.scores.append(0.0); self.masks.append(0)
                continue
            vals = dict(orc._values(rec))
            flag, score, alerts = orc.step(rec)
            mask = 0
            if orc.n_seen > orc.data_use_training:
                if combos is None:
                    for i, v in vals.items():
                        if v not in orc.known[i]:
                            mask |= 1 << i
                else:
                    n = len(orc.monitors)
                    for c, members in enumerate(combos):
                        if all(i in vals for i in members) and tuple(vals[i] for i in members) not in orc.known_combos[c]:
                            mask |= 1 << (n + c)
            assert bin(mask).count("1") == score and bool(mask) == flag
            self.flags.append(int(flag)); self.scores.append(float(score)); self.masks.append(mask)
            if flag:
                self.outputs.append(orc.make_output(rec, score, alerts).SerializeToString())
        return self


def new_run(config: dict, combo: bool = False, name: Optional[str] = None, clock=lambda: 1773848383) -> Run:
    if combo:
        return Run(NewValueComboDetectorOracle(name=name or "NewValueComboDetector", config=config, clock=clock))
    return Run(NewValueDetectorOracle(name=name or "NewValueDetector", config=config, clock=clock))
