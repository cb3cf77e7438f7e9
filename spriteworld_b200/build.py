"""Builds spriteworld_b200/csrc/libspriteworld_b200.so with nvcc for sm_90a (in-tree), and the
small host-side helper csrc/libswb_host.so (C, gcc: scene packing for the batched environment's
refill; optional -- without it the NumPy path runs).

    python -m spriteworld_b200.build [--force]
"""
import os
import shutil
import subprocess
import sys

CSRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'csrc')
LIB = os.path.join(CSRC, 'libspriteworld_b200.so')
SOURCES = ['swb_api.cu']
HEADERS = ['swb_device.cuh', 'swb_render.cuh', 'swb_sampler.cuh', 'swb_states.cuh', 'swb_step.cuh', 'swb_tables.h',
           os.path.join('..', '..', 'include', 'spriteworld_b200.h')]

NVCC_FLAGS = [
    '-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-lineinfo', '-std=c++17',
    # parity: the reference's float/double arithmetic is never FMA-contracted
    '-fmad=false',
    '-Xcompiler', '-fPIC', '-shared', '-lcudart',
]


def _nvcc():
  for cand in (os.environ.get('NVCC'), shutil.which('nvcc'), '/usr/local/cuda/bin/nvcc'):
    if cand and os.path.exists(cand):
      return cand
  raise RuntimeError('nvcc not found')


def is_stale():
  """True if the library is missing or older than its sources or this file (which holds the
  compiler flags, e.g. the target architecture)."""
  if not os.path.exists(LIB):
    return True
  t = os.path.getmtime(LIB)
  inputs = [os.path.join(CSRC, f) for f in SOURCES + HEADERS] + [os.path.abspath(__file__)]
  return any(os.path.getmtime(f) > t for f in inputs)


HOST_LIB = os.path.join(CSRC, 'libswb_host.so')
HOST_SRC = os.path.join(CSRC, 'swb_host_pack.c')
# parity with NumPy's elementwise float arithmetic: no contraction
HOST_FLAGS = ['-O3', '-ffp-contract=off', '-fPIC', '-shared', '-Wall', '-Wextra']


def build_host(force=False):
  """libswb_host.so (gcc).  Returns its path, or None if there is no C compiler."""
  if not force and os.path.exists(HOST_LIB) and os.path.getmtime(HOST_LIB) >= max(
      os.path.getmtime(HOST_SRC), os.path.getmtime(os.path.abspath(__file__))):
    return HOST_LIB
  cc = shutil.which('gcc') or shutil.which('cc')
  if not cc:
    return None
  proc = subprocess.run([cc] + HOST_FLAGS + ['-o', HOST_LIB, HOST_SRC], stdout=subprocess.PIPE,
                        stderr=subprocess.STDOUT, text=True)
  if proc.returncode:
    sys.stderr.write(proc.stdout)
    raise RuntimeError('building libswb_host.so failed (%d)' % proc.returncode)
  return HOST_LIB


SAMPLER_HOST_LIB = os.path.join(CSRC, 'libswb_sampler_host.so')
SAMPLER_HOST_SRC = os.path.join(CSRC, 'swb_sampler_host.cpp')
SAMPLER_HOST_INPUTS = [SAMPLER_HOST_SRC, os.path.join(CSRC, 'swb_sampler.cuh'),
                       os.path.join(CSRC, '..', '..', 'include', 'spriteworld_b200.h')]
# the same arithmetic as the kernels built with -fmad=false: no contraction
SAMPLER_HOST_FLAGS = ['-O2', '-std=c++17', '-ffp-contract=off', '-fPIC', '-shared', '-Wall', '-Wextra']


def build_sampler_host(force=False):
  """libswb_sampler_host.so (g++): the device scene sampler built for the CPU
  (scene_program.sample_on_host), the restatement the kernels are tested against."""
  if not force and os.path.exists(SAMPLER_HOST_LIB) and os.path.getmtime(SAMPLER_HOST_LIB) >= max(
      [os.path.getmtime(f) for f in SAMPLER_HOST_INPUTS] + [os.path.getmtime(os.path.abspath(__file__))]):
    return SAMPLER_HOST_LIB
  cxx = shutil.which('g++') or shutil.which('c++')
  if not cxx:
    raise RuntimeError('no C++ compiler for libswb_sampler_host.so')
  proc = subprocess.run([cxx] + SAMPLER_HOST_FLAGS + ['-o', SAMPLER_HOST_LIB, SAMPLER_HOST_SRC],
                        stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
  if proc.returncode:
    sys.stderr.write(proc.stdout)
    raise RuntimeError('building libswb_sampler_host.so failed (%d)' % proc.returncode)
  return SAMPLER_HOST_LIB


def build(force=False, verbose=False):
  build_host(force)
  build_sampler_host(force)
  if not force and not is_stale():
    return LIB
  cmd = [_nvcc()] + NVCC_FLAGS + (['-Xptxas', '-v'] if verbose else []) + ['-o', LIB] + SOURCES
  proc = subprocess.run(cmd, cwd=CSRC, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
  if verbose or proc.returncode:
    sys.stderr.write(proc.stdout)
  if proc.returncode:
    raise RuntimeError('nvcc failed (%d)' % proc.returncode)
  return LIB


if __name__ == '__main__':
  print(build(force='--force' in sys.argv, verbose='-v' in sys.argv))
