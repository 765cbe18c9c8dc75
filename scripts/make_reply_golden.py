#!/usr/bin/env python
"""Record tests/golden/component_replies.json.xz: every reply, n_alerts and n_seen of the scenarios of
tests/test_emu_reply_golden.py, run on the CPU emulator by the component of this tree.  Record it from a commit whose
replies are known to be right; the test then pins them for every later change.  scripts/make_reply_golden.py"""
import json
import lzma
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "tests"), ROOT]

import emu_harness  # noqa: E402
import test_emu_reply_golden as scenarios  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")


def main() -> None:
    replies = scenarios.record(emu_harness.lib(), GOLDEN)
    text = json.dumps(replies, indent=0, sort_keys=True)
    with lzma.open(os.path.join(GOLDEN, scenarios.FIXTURE), "wt", preset=9 | lzma.PRESET_EXTREME) as f:
        f.write(text)
    print("written:", scenarios.FIXTURE, len(replies), "scenarios,",
          sum(len(v) for v in replies.values()), "messages")


if __name__ == "__main__":
    main()
