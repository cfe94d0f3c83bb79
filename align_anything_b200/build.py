"""Build recipe for libaa_b200.so (hand-written sm_90a CUDA behind a C ABI).

    python -m align_anything_b200.build          # incremental
    python -m align_anything_b200.build --force

nvcc cross-compiles without a GPU.  The .so is written next to the sources (in-tree, git-ignored), where
_lib.py loads it from.
"""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
INCLUDE = os.path.join(os.path.dirname(HERE), 'include')
LIB = os.path.join(CSRC, 'libaa_b200.so')
OBJ_DIR = os.path.join(CSRC, 'build')
SOURCES = ['capi.cu', 'logprob.cu', 'logprob_fused.cu', 'dpo.cu', 'score_head.cu', 'ppo.cu', 'layout.cu', 'linear_logprob.cu', 'linear_backward.cu']
NVCC_FLAGS = [
    '-gencode', 'arch=compute_90a,code=sm_90a',
    '-O3', '-lineinfo', '-std=c++17',
    '-Xcompiler', '-fPIC',
    '-Xptxas', '-v',
    '--expt-relaxed-constexpr',
]


def _nvcc() -> str:
    cand = shutil.which('nvcc') or '/usr/local/cuda/bin/nvcc'
    if not os.path.exists(cand):
        raise RuntimeError('nvcc not found: libaa_b200.so cannot be built (there is no CPU fallback)')
    return cand


def _stamp() -> str:
    h = hashlib.sha256()
    for name in sorted(os.listdir(CSRC)):
        if name.endswith(('.cu', '.cuh')):
            with open(os.path.join(CSRC, name), 'rb') as f:
                h.update(name.encode())
                h.update(f.read())
    with open(os.path.join(INCLUDE, 'aa_b200.h'), 'rb') as f:
        h.update(f.read())
    h.update(' '.join(NVCC_FLAGS).encode())
    return h.hexdigest()


def is_fresh() -> bool:
    stamp_file = LIB + '.stamp'
    return os.path.exists(LIB) and os.path.exists(stamp_file) and open(stamp_file).read().strip() == _stamp()


def build_experiment(tag: str, defines: list[str]) -> str:
    """Build a side copy libaa_b200.<tag>.so with extra -D flags (tuning experiments only; select it
    at run time with AA_B200_LIB=<path>)."""
    nvcc = _nvcc()
    out = os.path.join(CSRC, f'libaa_b200.{tag}.so')
    srcs = [os.path.join(CSRC, s) for s in SOURCES]
    flags = [f for f in NVCC_FLAGS if f not in ('-Xptxas', '-v')]
    cmd = [nvcc, *flags, *[f'-D{d}' for d in defines], '-I', INCLUDE, '-shared', '-o', out, *srcs]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f'nvcc failed:\n{r.stdout}\n{r.stderr}')
    return out


def build(force: bool = False, verbose: bool = False) -> str:
    """Compile every .cu for sm_90a and link libaa_b200.so.  Returns the library path."""
    if not force and is_fresh():
        return LIB
    nvcc = _nvcc()
    os.makedirs(OBJ_DIR, exist_ok=True)
    logs = {}

    def compile_one(src):
        obj = os.path.join(OBJ_DIR, src.replace('.cu', '.o'))
        cmd = [nvcc, *NVCC_FLAGS, '-I', INCLUDE, '-c', os.path.join(CSRC, src), '-o', obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        logs[src] = r.stderr
        if r.returncode != 0:
            raise RuntimeError(f'nvcc failed on {src}:\n{r.stdout}\n{r.stderr}')
        return obj

    with ThreadPoolExecutor(max_workers=min(8, len(SOURCES))) as ex:
        objs = list(ex.map(compile_one, SOURCES))
    cmd = [nvcc, '-gencode', 'arch=compute_90a,code=sm_90a', '-shared', '-o', LIB, *objs]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f'link failed:\n{r.stdout}\n{r.stderr}')
    with open(LIB + '.stamp', 'w') as f:
        f.write(_stamp())
    with open(os.path.join(OBJ_DIR, 'ptxas.log'), 'w') as f:
        for src in SOURCES:
            f.write(f'==== {src} ====\n{logs.get(src, "")}\n')
    if verbose:
        for src in SOURCES:
            print(f'==== {src} ====\n{logs.get(src, "")}')
    return LIB


if __name__ == '__main__':
    path = build(force='--force' in sys.argv, verbose='-v' in sys.argv)
    print(path)
