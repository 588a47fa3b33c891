"""Builds libmpengine.so (the CUDA engine + C ABI) in-tree for sm_90a (H100)."""

from __future__ import annotations

import os
import shutil
import subprocess

_HERE = os.path.dirname(os.path.abspath(__file__))
SOURCES = ['engine.cu']
HEADERS = ['common.cuh', 'family_load.h', 'render.cuh', 'step_common.cuh', 'step_clean_up.cuh', 'step_commons.cuh', 'step_territory.cuh', 'step_coins.cuh', 'step_mining.cuh', 'state_bank.cuh']
LIB_PATH = os.path.join(_HERE, 'libmpengine.so')

NVCC_FLAGS = [
    '-gencode', 'arch=compute_90a,code=sm_90a', '-lineinfo', '-O3',
    '-std=c++17', '--fmad=false', '-shared', '-Xcompiler', '-fPIC',
]


def _nvcc() -> str:
  for cand in (shutil.which('nvcc'), '/usr/local/cuda/bin/nvcc'):
    if cand and os.path.exists(cand):
      return cand
  raise FileNotFoundError('nvcc not found')


def is_stale() -> bool:
  if not os.path.exists(LIB_PATH):
    return True
  built = os.path.getmtime(LIB_PATH)
  deps = [os.path.join(_HERE, 'csrc', f) for f in SOURCES + HEADERS]
  root = os.path.dirname(_HERE)
  deps += [os.path.join(root, 'include', 'mp_engine.h'),
           os.path.join(root, 'include', 'mpb_format.h')]
  return any(os.path.getmtime(d) > built for d in deps if os.path.exists(d))


def build(force: bool = False, verbose: bool = False) -> str:
  """Compiles the engine if sources are newer than the library."""
  if not force and not is_stale():
    return LIB_PATH
  cmd = [_nvcc()] + NVCC_FLAGS
  if verbose:
    cmd += ['-Xptxas', '-v']
  cmd += ['-o', LIB_PATH] + [os.path.join(_HERE, 'csrc', s) for s in SOURCES]
  subprocess.check_call(cmd)
  return LIB_PATH


if __name__ == '__main__':
  print(build(force=True, verbose=True))
