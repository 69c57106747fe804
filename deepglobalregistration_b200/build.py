"""Build libdgr_b200.so in-tree with nvcc for sm_90a (no torch headers in the ABI, so a
full rebuild takes well under a minute and needs no GPU).

    python -m deepglobalregistration_b200.build [--force]
"""
import hashlib
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, 'csrc')
INCLUDE = os.path.join(ROOT, 'include')
LIB = os.path.join(HERE, 'libdgr_b200.so')
OBJ_DIR = os.path.join(HERE, 'build')

NVCC_FLAGS = ['-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-lineinfo', '-std=c++17',
              '-Xcompiler', '-fPIC', '--expt-relaxed-constexpr', '-I', INCLUDE, '-I', CSRC]
NVCC_FLAGS += os.environ.get('DGR_EXTRA_NVCC_FLAGS', '').split()      # extra build flags (A/B experiments)


def _nvcc():
  for cand in (os.environ.get('NVCC'), '/usr/local/cuda/bin/nvcc', 'nvcc'):
    if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
      return cand
  raise RuntimeError('nvcc not found')


def sources():
  return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith('.cu'))


def _fingerprint():
  h = hashlib.sha256()
  for d in (CSRC, INCLUDE):
    for f in sorted(os.listdir(d)):
      with open(os.path.join(d, f), 'rb') as fh:
        h.update(f.encode())
        h.update(fh.read())
  h.update(' '.join(NVCC_FLAGS).encode())
  return h.hexdigest()


def build(force=False, verbose=False):
  """Compile every csrc/*.cu for sm_90a and link libdgr_b200.so.  Returns its path."""
  os.makedirs(OBJ_DIR, exist_ok=True)
  stamp = os.path.join(OBJ_DIR, 'fingerprint')
  fp = _fingerprint()
  if not force and os.path.exists(LIB) and os.path.exists(stamp) and open(stamp).read() == fp:
    return LIB
  nvcc = _nvcc()
  flags = NVCC_FLAGS + (['-Xptxas', '-v'] if verbose else [])

  def compile_one(src):
    obj = os.path.join(OBJ_DIR, os.path.basename(src)[:-3] + '.o')
    r = subprocess.run([nvcc] + flags + ['-c', src, '-o', obj], capture_output=True, text=True)
    return src, obj, r

  with ThreadPoolExecutor(max_workers=8) as ex:
    results = list(ex.map(compile_one, sources()))
  objs = []
  for src, obj, r in results:
    if verbose or r.returncode != 0:
      sys.stderr.write(r.stdout + r.stderr)
    if r.returncode != 0:
      raise RuntimeError(f'nvcc failed on {src}')
    objs.append(obj)
  r = subprocess.run([nvcc, '-shared', '-o', LIB] + objs + ['-lcudart'], capture_output=True, text=True)
  if r.returncode != 0:
    sys.stderr.write(r.stdout + r.stderr)
    raise RuntimeError('link failed')
  with open(stamp, 'w') as fh:
    fh.write(fp)
  return LIB


if __name__ == '__main__':
  print(build(force='--force' in sys.argv, verbose='-v' in sys.argv))
