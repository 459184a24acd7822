"""Run a snippet of test code in a fresh Python interpreter -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

The kernel-launch checks trace with torch.profiler (CUPTI activity tracing).  CUPTI keeps process-wide state, and
late in a long test process a trace can come back without some of its kernel records (a forward trace once held the
gate GEMM but not the split kernel launched just before it).  Those checks therefore trace in a child interpreter
whose profiler has not been used before, and the test process's profiler stays untouched."""
import json
import os
import subprocess
import sys

TESTS = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(TESTS)
TAG = "RESULT "


def run_json(code, *args, timeout=600):
    """Run `code` in a fresh interpreter with tests/ and the repository root first on sys.path, sys.argv[1:] = args
    and the RGCN_* environment knobs cleared; the code prints one line `RESULT <json>`, which is returned decoded."""
    env = {k: v for k, v in os.environ.items() if not k.startswith("RGCN_")}
    flags = ["-s"] if sys.flags.no_user_site else []
    prologue = "import sys\nsys.path[:0] = [%r, %r]\n" % (TESTS, ROOT)
    p = subprocess.run([sys.executable] + flags + ["-c", prologue + code] + [str(a) for a in args],
                       capture_output=True, text=True, env=env, timeout=timeout)
    lines = [l for l in p.stdout.splitlines() if l.startswith(TAG)]
    assert p.returncode == 0 and lines, p.stdout[-2000:] + p.stderr[-4000:]
    return json.loads(lines[-1][len(TAG):])
