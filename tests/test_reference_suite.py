"""The reference's OWN test-suite (everything but tests/library_integration, which needs the
un-vendored detectmatelibrary components) run against this repo's stand-ins for the two
packages that cannot be installed offline: `pynng` (SP/PAIR0 transport) and the two
`detectmatelibrary` base modules.  The reference service and its tests are taken from
oracle/_ref, where `make -C oracle ref` (run by build()) copies them.

Bar: 0 failures, 0 collection errors.
"""
import os
import subprocess
import sys

import pytest

from oracle.ref_engine import REF_DIR

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.skipif(not os.path.isdir(os.path.join(REF_DIR, "tests")), reason="the reference is not in oracle/_ref (make -C oracle ref)")
def test_reference_suite_passes_on_the_shims(tmp_path, ipc_dir):
    shims = os.path.join(ROOT, "detectmateservice_b200", "shims")
    tests = os.path.join(REF_DIR, "tests")
    env = dict(os.environ)
    env["PYTHONPATH"] = os.pathsep.join([REF_DIR, shims, env.get("PYTHONPATH", "")])
    env.pop("DM_KERNEL", None)
    # the reference's tests put ipc:// sockets under their tmp_path: keep it short (107-byte socket paths)
    cmd = [sys.executable, "-m", "pytest", tests, "-q", "-x", "-p", "no:cacheprovider",
           "--ignore", os.path.join(tests, "library_integration"), "--rootdir", str(tmp_path),
           "--basetemp", os.path.join(ipc_dir, "t"), "--timeout", "120"]
    res = subprocess.run(cmd, cwd=str(tmp_path), env=env, capture_output=True, text=True, timeout=1500)
    tail = "\n".join((res.stdout + res.stderr).splitlines()[-40:])
    assert res.returncode == 0, "reference suite on the shims:\n" + tail
    assert " passed" in res.stdout and "error" not in res.stdout.splitlines()[-1].lower(), tail
