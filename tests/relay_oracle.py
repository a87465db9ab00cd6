"""TEST INFRASTRUCTURE — ctypes binding of the recursion relay's CPU oracle (tests/native/relay_oracle.cpp).

The library is compiled on first use into the temporary directory (keyed by a hash of its sources), so that neither the
tests nor tools/relay_bench.py write into the tree.  The product (binder_b200/) never imports this.
"""
import ctypes
import hashlib
import os
import shutil
import subprocess
import tempfile

import numpy as np

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_SRCS = [os.path.join(_ROOT, 'tests', 'native', 'relay_oracle.cpp'), os.path.join(_ROOT, 'oracle', 'oracle.cpp')]
_lib = None


def build():
    """Path of the compiled library, building it when its sources changed."""
    h = hashlib.sha256()
    for s in _SRCS:
        h.update(open(s, 'rb').read())
    so = os.path.join(tempfile.gettempdir(), 'binder_b200_relay_oracle_%s_%d.so' % (h.hexdigest()[:16], os.getuid()))
    if not os.path.exists(so):
        cxx = shutil.which(os.environ.get('CXX', 'g++')) or 'g++'
        tmp = '%s.%d.tmp' % (so, os.getpid())
        subprocess.check_call([cxx, '-O2', '-std=c++17', '-fPIC', '-pthread', '-shared', '-o', tmp, _SRCS[0]])
        os.replace(tmp, so)
    return so


def lib():
    global _lib
    if _lib is None:
        L = ctypes.CDLL(build())
        L.orc_relay_batch.argtypes = [ctypes.c_void_p] * 4 + [ctypes.c_uint32, ctypes.c_uint32, ctypes.c_void_p, ctypes.c_uint64,
                                                               ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int]
        _lib = L
    return _lib


def relay_batch(q_data, q_off, up_data, up_off, tcp=False, nthreads=1):
    """lib/recursion.js:287-327 on a batch: query i with upstream response i (empty = the lookup failed).
    Same call shape as Engine.relay_batch -> (out uint8[total], out_off uint32[n+1], out_len uint16[n], status uint8[n])."""
    q_data = np.ascontiguousarray(q_data, dtype=np.uint8)
    q_off = np.ascontiguousarray(q_off, dtype=np.uint32)
    up_data = np.ascontiguousarray(up_data, dtype=np.uint8)
    up_off = np.ascontiguousarray(up_off, dtype=np.uint32)
    n = len(q_off) - 1
    assert len(up_off) == n + 1
    out_cap = max(1, n * (65535 if tcp else 1200))
    out = np.empty(out_cap, dtype=np.uint8)
    out_off = np.zeros(n + 1, dtype=np.uint32)
    status = np.zeros(max(n, 1), dtype=np.uint8)
    rc = lib().orc_relay_batch(q_data.ctypes.data, q_off.ctypes.data, up_data.ctypes.data, up_off.ctypes.data, n,
                               1 if tcp else 0, out.ctypes.data, out_cap, out_off.ctypes.data, status.ctypes.data, nthreads)
    if rc != 0:
        raise RuntimeError('relay oracle failed (%d)' % rc)
    lens = np.diff(out_off.astype(np.int64)).astype(np.uint16)
    return out[:out_off[n]].copy(), out_off, lens, status[:n]


class RelayOracle(object):
    """A resolver-shaped object for binder_b200.recursion.Recursion: relay_batch on the CPU."""

    def relay_batch(self, q_data, q_off, up_data, up_off, tcp=False):
        return relay_batch(q_data, q_off, up_data, up_off, tcp)
