"""In-tree nvcc build of the C-ABI library ``libscoresde_b200.so`` for sm_90a.

No torch headers are involved: the library is plain CUDA C++ behind ``extern "C"``
entry points (``include/scoresde_b200.h``) and is loaded with ``ctypes``.  The
``.so`` is written next to this file so it travels with the repository snapshot.
"""
import hashlib
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
LIB = os.path.join(HERE, 'libscoresde_b200.so')
STAMP = os.path.join(HERE, '.libscoresde_b200.stamp')
SOURCES = ['api.cu', 'elementwise.cu', 'conv_simt.cu', 'conv_lowc.cu', 'gemm_tc.cu', 'attn_tc.cu', 'attn_flash.cu', 'pc_update.cu', 'engine.cu', 'ode.cu', 'losses.cu', 'tangent.cu']
NVCC_FLAGS = ['-gencode', 'arch=compute_90a,code=sm_90a', '-lineinfo', '-O3', '-std=c++17',
              '-Xcompiler', '-fPIC,-fvisibility=hidden', '--expt-relaxed-constexpr']


def _nvcc():
  for cand in (os.environ.get('NVCC'), shutil.which('nvcc'), '/usr/local/cuda/bin/nvcc'):
    if cand and os.path.exists(cand):
      return cand
  raise RuntimeError('nvcc not found: the CUDA path of score_sde_pytorch_b200 cannot be built')


def _digest():
  h = hashlib.sha256()
  files = sorted(os.listdir(CSRC)) + ['../../include/scoresde_b200.h']
  for f in files:
    p = os.path.join(CSRC, f)
    if os.path.isfile(p):
      h.update(f.encode())
      with open(p, 'rb') as fh:
        h.update(fh.read())
  h.update(' '.join(NVCC_FLAGS).encode())
  return h.hexdigest()


def build(force=False, verbose=False):
  """Compile every CUDA translation unit for sm_90a and link the shared library.
  Returns the library path.  Skips the work when sources are unchanged."""
  digest = _digest()
  if not force and os.path.exists(LIB) and os.path.exists(STAMP):
    with open(STAMP) as fh:
      if fh.read().strip() == digest:
        return LIB
  nvcc = _nvcc()
  objdir = os.path.join(HERE, 'build')
  os.makedirs(objdir, exist_ok=True)
  procs = []
  for src in SOURCES:
    obj = os.path.join(objdir, src.replace('.cu', '.o'))
    cmd = [nvcc] + NVCC_FLAGS + (['-Xptxas', '-v'] if verbose else []) + ['-c', os.path.join(CSRC, src), '-o', obj]
    procs.append((src, obj, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
  objs = []
  for src, obj, p in procs:
    out, _ = p.communicate()
    if p.returncode != 0:
      raise RuntimeError(f'nvcc failed on {src}:\n{out}')
    if verbose:
      print(out)
    objs.append(obj)
  cmd = [nvcc, '-shared', '-gencode', 'arch=compute_90a,code=sm_90a', '-o', LIB] + objs
  r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
  if r.returncode != 0:
    raise RuntimeError(f'link failed:\n{r.stdout}')
  with open(STAMP, 'w') as fh:
    fh.write(digest)
  return LIB


if __name__ == '__main__':
  print(build(force='--force' in sys.argv, verbose='-v' in sys.argv))
