"""Builds binder_b200/libbinder_b200.so (CUDA kernels for sm_90a + the C ABI) in-tree.

    python -m binder_b200.build [--force]
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
SO = os.path.join(HERE, 'libbinder_b200.so')
SRCS = [os.path.join(HERE, 'csrc', f) for f in ('engine.cu', 'zone_build.cpp', 'balancer_frames.cpp', 'balancer_relay.cpp',
                                                'balancer_tcp.cpp', 'balancer_query_log.cpp')]
DEPS = SRCS + [os.path.join(HERE, 'csrc', 'zone_image.h'), os.path.join(HERE, 'csrc', 'resolve_device.cuh'),
               os.path.join(HERE, 'csrc', 'balancer_backend.h'), os.path.join(HERE, 'csrc', 'relay_device.cuh'), os.path.join(HERE, 'csrc', 'log_device.cuh'),
               os.path.join(HERE, 'csrc', 'forward_device.cuh'),
               os.path.join(os.path.dirname(HERE), 'include', 'binder_b200.h')]
NVCC = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
FLAGS = ['-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-lineinfo', '-std=c++17',
         '-Xcompiler', '-fPIC,-Wall,-Wno-unused-function', '-shared', '-cudart', 'static']


def up_to_date():
    return os.path.exists(SO) and all(os.path.getmtime(SO) >= os.path.getmtime(d) for d in DEPS)


def build(force=False, verbose=False):
    if not force and up_to_date():
        return SO
    extra = os.environ.get('BB_NVCC_DEFINES', '').split()      # e.g. -DBB_MIN_BLOCKS=6 (tuning experiments)
    cmd = [NVCC] + FLAGS + extra + (['-Xptxas', '-v'] if verbose else []) + ['-o', SO] + SRCS
    subprocess.check_call(cmd)
    return SO


if __name__ == '__main__':
    print(build(force='--force' in sys.argv, verbose='-v' in sys.argv))
