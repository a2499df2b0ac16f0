"""In-tree build of librigl_b200.so (nvcc, sm_90a only).

  python -m rigl_b200.build [--force] [--verbose]

The library is the C-ABI of include/rigl_b200.h; it links cudart statically and
resolves the driver API (cuTensorMapEncodeTiled) at run time through
cudaGetDriverEntryPoint, so it loads on a machine without libcuda (CPU tests
check the exported symbols there).
"""
import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
ROOT = os.path.dirname(HERE)
LIB = os.path.join(HERE, 'librigl_b200.so')
STAMP = os.path.join(HERE, 'build', 'stamp.txt')

NVCC_FLAGS = [
    '-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-std=c++17', '-lineinfo',
    '-Xcompiler', '-fPIC', '-Xcompiler', '-fvisibility=hidden', '--expt-relaxed-constexpr',
    '-cudart', 'static',
]


def sources():
  return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith('.cu'))


def _digest():
  h = hashlib.sha256()
  for p in sources() + sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(('.cuh', '.h'))) + \
      [os.path.join(ROOT, 'include', 'rigl_b200.h')]:
    h.update(p.encode())
    with open(p, 'rb') as f:
      h.update(f.read())
  h.update(' '.join(NVCC_FLAGS).encode())
  return h.hexdigest()


def nvcc_path():
  for cand in (os.environ.get('NVCC'), '/usr/local/cuda/bin/nvcc', 'nvcc'):
    if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
      return cand
  return 'nvcc'


def build(force=False, verbose=False):
  """Compiles every .cu under csrc/ into one shared library.  Returns its path."""
  digest = _digest()
  if not force and os.path.exists(LIB) and os.path.exists(STAMP):
    with open(STAMP) as f:
      if f.read().strip() == digest:
        return LIB
  os.makedirs(os.path.join(HERE, 'build'), exist_ok=True)
  objs = []
  procs = []
  for src in sources():
    obj = os.path.join(HERE, 'build', os.path.basename(src)[:-3] + '.o')
    cmd = [nvcc_path()] + NVCC_FLAGS + (['-Xptxas', '-v'] if verbose else []) + ['-c', src, '-o', obj]
    procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    objs.append(obj)
  failed = False
  for src, p in procs:
    out, _ = p.communicate()
    if p.returncode != 0 or verbose:
      sys.stderr.write('--- nvcc %s\n%s\n' % (os.path.basename(src), out))
    failed = failed or p.returncode != 0
  if failed:
    raise RuntimeError('nvcc failed building librigl_b200.so')
  tmp = LIB + '.tmp.%d' % os.getpid()       # link aside, then rename: a concurrent reader never sees a partial file
  link = [nvcc_path(), '-shared', '-o', tmp] + objs + ['-cudart', 'static', '-Xcompiler', '-fPIC']
  r = subprocess.run(link, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
  if r.returncode != 0:
    raise RuntimeError('link failed:\n' + r.stdout)
  os.replace(tmp, LIB)
  with open(STAMP, 'w') as f:
    f.write(digest)
  return LIB


if __name__ == '__main__':
  print(build(force='--force' in sys.argv, verbose='--verbose' in sys.argv))
