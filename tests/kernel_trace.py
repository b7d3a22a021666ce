"""What a call runs on the GPU, read from torch.profiler in a process of its own.

`trace(builder, cases, per_process)` runs each case in a child process (`sys.executable -s`, with tests/ and the
repository root on its path), `per_process` cases per child, so that no profiler session can disturb the tests that
follow.  `builder` is "module:function"; `function(*case)` builds the case's inputs and returns a zero-argument callable
(one that returns an int is a C ABI entry and must return 0).  For each case the child calls it once outside any
profiler session (module load, descriptors), then profiles one more call, up to five times: a profiler session on a
shared GPU occasionally records no CUDA activity at all.  The case's `Record` holds the change of launch_count() around
the profiled call and every kernel, copy and fill the session recorded, in timestamp order, as `Event`s."""
import collections
import importlib
import json
import os
import re
import subprocess
import sys
import tempfile
import time
import typing

import torch

TESTS = os.path.dirname(os.path.abspath(__file__))
CATEGORIES = ("kernel", "gpu_memcpy", "gpu_memset")
PAD_S = 0.02   # idle seconds before and after the profiled call, inside the session
Event = collections.namedtuple("Event", "cat name grid smem")   # grid and shared memory are None for copies and fills


class Record(typing.NamedTuple):
    launches: int
    events: list

    @property
    def names(self):
        return [e.name for e in self.events]


def trace(builder, cases, per_process, env=None):
    """One Record per case (see the module docstring); `env` is added to the child's environment."""
    cases = [list(c) for c in cases]
    out = []
    for i in range(0, len(cases), per_process):
        r = subprocess.run([sys.executable, "-s", __file__, builder, json.dumps(cases[i:i + per_process])],
                           capture_output=True, text=True, timeout=900, env=dict(os.environ, **(env or {})))
        assert r.returncode == 0, r.stderr[-3000:]
        out += [Record(n, [Event(*e) for e in ev]) for n, ev in json.loads(r.stdout.strip().splitlines()[-1])]
    return out


def short_names(names):
    """The W4A16 kernels among `names` as `w4a16_<name>_kernel`, or `w4a16_wgmma_kernel<TN>` (TN is the wgmma kernel's
    last template argument)."""
    found = set()
    for name in names:
        mt = re.search(r"w4a16_(\w+?)_kernel(<[^>]*?(\d+)>)?", name)
        if mt:
            found.add(f"w4a16_wgmma_kernel<{mt.group(3)}>" if mt.group(1) == "wgmma" else f"w4a16_{mt.group(1)}_kernel")
    return found


def _check_rc(rc):
    assert not isinstance(rc, int) or rc == 0, f"return code {rc}"


def _events(prof):
    fd, path = tempfile.mkstemp(suffix=".json")
    os.close(fd)
    try:
        prof.export_chrome_trace(path)
        with open(path) as f:
            events = json.load(f)["traceEvents"]
    finally:
        os.unlink(path)
    events = sorted((e for e in events if e.get("cat") in CATEGORIES), key=lambda e: e.get("ts", 0))
    return [[e["cat"], e["name"], e.get("args", {}).get("grid"), e.get("args", {}).get("shared memory")]
            for e in events]


def _child(builder, cases):
    import llm_awq_b200 as P   # after __main__ has put the repository root on the path
    mod, fn = builder.split(":")
    build = getattr(importlib.import_module(mod), fn)
    eng = P.engine()
    out = []
    for case in cases:
        call = build(*case)
        _check_rc(call())
        torch.cuda.synchronize()
        for _ in range(5):
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                # GPU records outside the session's capture window are dropped, and the window is on the host clock:
                # margins keep a call of a few microseconds inside it when the two clocks disagree slightly
                time.sleep(PAD_S)
                c0 = eng.launch_count()
                _check_rc(call())
                torch.cuda.synchronize()
                launches = eng.launch_count() - c0
                time.sleep(PAD_S)
            events = _events(prof)
            if events:
                break
        out.append([launches, events])
    print(json.dumps(out))


if __name__ == "__main__":
    sys.path.insert(0, os.path.dirname(TESTS))
    _child(sys.argv[1], json.loads(sys.argv[2]))
