"""Which CUDA kernels a call launches, seen through torch.profiler (CUPTI): for tests that pin the launch path a shape,
dtype or layout selects.  Kernel names come demangled, e.g. ``void (anonymous namespace)::dwconv2d_fwd_kernel<float,
true, 4>((anonymous namespace)::DwArgs)``; ``targs`` splits out the template arguments.

Once a process has run the profiler, a fork of it (the multi-process and subprocess tests of the suite fork) can leave
later sessions of that process without kernel records.  ``in_child`` therefore runs a module's captures in a fresh
interpreter of their own and hands the names back; the parity checks stay in the test process."""
import json
import os
import re
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def targs(name, prefix):
    """Template arguments of the instance ``name`` whose name ends with ``prefix`` (e.g. ``"dwconv2d_fwd_kernel<"``)."""
    body = name[name.index(prefix) + len(prefix):]
    depth, args, cur = 1, [], ""
    for ch in body:
        depth += ch == "<"
        depth -= ch == ">"
        if depth == 0 or (depth == 1 and ch == ","):
            args.append(cur.strip())
            cur = ""
            if depth == 0:
                return args
        else:
            cur += ch
    raise AssertionError(f"unterminated template arguments in {name!r}")


def launched(fn, pattern):
    """-> (fn(), names of the kernels matching ``pattern`` (a regex) that ran during the call)."""
    rx = re.compile(pattern) if isinstance(pattern, str) else pattern
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        res = fn()
        torch.cuda.synchronize()
    return res, [e.name for e in prof.events() if rx.search(e.name)]


def retry(run, complete, tries=6, pause=0.25):
    """Now and then a short profiler session loses kernel records, sometimes several sessions in a row: ``run()`` is taken
    again, up to ``tries`` times in all, until ``complete(result)`` holds, waiting ``pause`` seconds times the number of
    failed tries before each new one so that a burst of lost records can pass.  A complete first capture costs nothing
    extra.  The last result is returned either way, so a wrong launch still fails the caller."""
    for i in range(tries):
        if i:
            time.sleep(pause * i)
        res = run()
        if complete(res):
            break
    return res


def names_of(fn, pattern, n=1):
    """Names of the kernels matching ``pattern`` that ``fn()`` launches, taken again while fewer than ``n`` were seen."""
    return retry(lambda: launched(fn, pattern), lambda r: len(r[1]) >= n)[1]


def in_child(func):
    """The JSON result of ``func()`` ("module:function", run from the repository root) computed in a fresh interpreter."""
    mod, name = func.split(":")
    code = f"import json, sys\nfrom {mod} import {name}\nsys.stdout.write('\\n' + json.dumps({name}()) + '\\n')"
    p = subprocess.run([sys.executable, "-c", code], cwd=ROOT, capture_output=True, text=True, timeout=1200)
    assert p.returncode == 0, p.stdout[-3000:] + p.stderr[-3000:]
    return json.loads(p.stdout.strip().splitlines()[-1])
