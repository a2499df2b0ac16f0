"""Runs test cases in a fresh interpreter, under a given environment and with a time limit.

The library reads its RIGL_* switches once per process, so a test of a kernel variant that only an environment
variable selects has to run in a child process.  The child is given a timeout: a pipeline that never completes
(a producer and its consumers that disagree on which stages they fill) then fails its test instead of blocking
the suite.  Each call runs under torch.profiler (CUDA activity only), and the names of the kernels it launched
come back to the caller, so a variant test can check that the kernel it exists for actually ran.
"""
import json
import os
import re
import subprocess
import sys

import pytest

TESTS = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(TESTS)
_RESULT = 'ISOLATED_KERNELS '

_CHILD = r'''
import importlib, json, sys
sys.path[:0] = [%(root)r, %(tests)r]
import torch
from torch.autograd import DeviceType
from torch.profiler import ProfilerActivity, profile
mod = importlib.import_module(%(module)r)
ran = []
for fn, args in %(calls)r:
  print('running %%s%%r' %% (fn, args), flush=True)
  with profile(activities=[ProfilerActivity.CUDA]) as prof:
    getattr(mod, fn)(*args)
    torch.cuda.synchronize()
  ran.append(sorted({e.name for e in prof.events() if e.device_type == DeviceType.CUDA}))
print(%(result)r + json.dumps(ran), flush=True)
'''


def run_isolated(module, calls, env=None, timeout=300):
  """Runs `module.fn(*args)` for every `(fn, args)` of `calls`, in order, in one child interpreter whose
  environment is ours plus `env`.  `args` must be literals (they travel as their repr).  Returns one list per call:
  the names of the CUDA kernels (and memsets / copies) the call launched.  Fails the calling test when a call
  raises, the child dies, or it has not finished after `timeout` seconds (the child is then killed)."""
  code = _CHILD % dict(root=ROOT, tests=TESTS, module=module, calls=[(fn, tuple(args)) for fn, args in calls],
                       result=_RESULT)
  cmd = [sys.executable] + (['-s'] if sys.flags.no_user_site else []) + ['-c', code]
  try:
    out = subprocess.run(cmd, env=dict(os.environ, **(env or {})), stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                         text=True, timeout=timeout)
  except subprocess.TimeoutExpired as e:
    tail = e.stdout.decode(errors='replace') if isinstance(e.stdout, bytes) else (e.stdout or '')
    pytest.fail('%s under %r did not finish within %d s (killed); last output:\n%s' % (module, env, timeout,
                                                                                     tail[-3000:]))
  lines = [l for l in out.stdout.splitlines() if l.startswith(_RESULT)]
  if out.returncode != 0 or not lines:
    pytest.fail('%s under %r failed (exit code %d):\n%s' % (module, env, out.returncode, out.stdout[-3000:]))
  ran = json.loads(lines[-1][len(_RESULT):])
  assert len(ran) == len(calls)
  return ran


def assert_ran(names, pattern, what):
  """Some kernel name in `names` matches the regular expression `pattern`."""
  assert any(re.search(pattern, n) for n in names), '%s: no kernel matching %r ran; ran: %s' % (what, pattern, names)


def assert_not_ran(names, pattern, what):
  hits = [n for n in names if re.search(pattern, n)]
  assert not hits, '%s: %r should not run; ran: %s' % (what, pattern, hits)
