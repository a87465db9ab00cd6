"""TEST INFRASTRUCTURE — ctypes binding of the recursion forward / match CPU oracle (tests/native/forward_oracle.cpp).

Compiled on first use into the temporary directory (keyed by a hash of its sources), like tests/relay_oracle.py.  The
product (binder_b200/) never imports this.  ForwardOracle is an Engine-shaped stand-in for binder_b200.forward.GpuRecursion.
"""
import ctypes
import hashlib
import os
import shutil
import subprocess
import tempfile

import numpy as np

import relay_oracle
from binder_b200.engine import FORWARD_ROUTES, ip_u32

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_SRCS = [os.path.join(_ROOT, 'tests', 'native', 'forward_oracle.cpp'), os.path.join(_ROOT, 'oracle', 'oracle.cpp')]
_lib = None


def build():
    h = hashlib.sha256()
    for s in _SRCS:
        h.update(open(s, 'rb').read())
    so = os.path.join(tempfile.gettempdir(), 'binder_b200_forward_oracle_%s_%d.so' % (h.hexdigest()[:16], os.getuid()))
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
        P, U32, U64 = ctypes.c_void_p, ctypes.c_uint32, ctypes.c_uint64
        L.orc_fwd_id.argtypes = [U64, U32, ctypes.c_int]
        L.orc_fwd_id.restype = U32
        L.orc_forward_batch.argtypes = [ctypes.c_char_p, P, U32, P, P, P, U32, P, P, U32, U64, P, P, P, P, P]
        L.orc_match.argtypes = [ctypes.c_char_p, P, U32, P, P, P, U32, P, P, P, P, U32, P, P, P, U32, U64, P, P]
        _lib = L
    return _lib


def fwd_id(key, j, inverse=False):
    return int(lib().orc_fwd_id(key & (2 ** 64 - 1), j, 1 if inverse else 0))


class Table(object):
    """The filter (region domain, datacenter names) and the upstream table [(ip, port, dc index)]."""

    def __init__(self, region, dcs, upstreams):
        self.region, self.dcs, self.upstreams = region, list(dcs), list(upstreams)
        self._names = [d.encode('latin-1') for d in self.dcs]
        self._dcs = (ctypes.c_char_p * max(len(self.dcs), 1))(*self._names)
        self._ip = np.array([ip_u32(a) for a, _, _ in self.upstreams] or [0], dtype=np.uint32)
        self._port = np.array([p for _, p, _ in self.upstreams] or [0], dtype=np.uint16)
        self._dc = np.array([d for _, _, d in self.upstreams] or [0], dtype=np.uint8)

    def args(self):
        return (self.region.encode('latin-1'), ctypes.cast(self._dcs, ctypes.c_void_p), len(self.dcs), self._ip.ctypes.data,
                self._port.ctypes.data, self._dc.ctypes.data, len(self.upstreams))


def forward_batch(table, data, off, key):
    """Same call shape and results as Engine.forward_batch."""
    data = np.ascontiguousarray(data, dtype=np.uint8)
    off = np.ascontiguousarray(off, dtype=np.uint32)
    n = len(off) - 1
    uq = np.zeros(max(int(off[n]), 16), dtype=np.uint8)
    uq_off = np.zeros(n + 1, dtype=np.uint32)
    order = np.zeros(max(n, 1), dtype=np.uint32)
    group_off = np.zeros(FORWARD_ROUTES + 1, dtype=np.uint32)
    route = np.zeros(max(n, 1), dtype=np.uint8)
    lib().orc_forward_batch(*table.args(), data.ctypes.data, off.ctypes.data, n, key & (2 ** 64 - 1), uq.ctypes.data,
                            uq_off.ctypes.data, order.ctypes.data, group_off.ctypes.data, route.ctypes.data)
    return uq[:uq_off[n]].copy(), uq_off, order[:n], group_off, route[:n]


def match_upstreams(table, resp, resp_off, src_ip, src_port, q_data, q_off, route, key):
    """Same call shape and results as Engine.match_upstreams."""
    resp = np.ascontiguousarray(resp, dtype=np.uint8)
    resp_off = np.ascontiguousarray(resp_off, dtype=np.uint32)
    src_ip = np.ascontiguousarray(src_ip, dtype=np.uint32)
    src_port = np.ascontiguousarray(src_port, dtype=np.uint16)
    q_data = np.ascontiguousarray(q_data, dtype=np.uint8)
    q_off = np.ascontiguousarray(q_off, dtype=np.uint32)
    route = np.ascontiguousarray(route, dtype=np.uint8)
    n_resp, n = len(resp_off) - 1, len(q_off) - 1
    up = np.zeros(max(int(resp_off[n_resp]), 16), dtype=np.uint8)
    up_off = np.zeros(n + 1, dtype=np.uint32)
    lib().orc_match(*table.args(), resp.ctypes.data, resp_off.ctypes.data, src_ip.ctypes.data, src_port.ctypes.data, n_resp,
                    q_data.ctypes.data, q_off.ctypes.data, route.ctypes.data, n, key & (2 ** 64 - 1), up.ctypes.data, up_off.ctypes.data)
    return up[:up_off[n]].copy(), up_off


class ForwardOracle(object):
    """An Engine-shaped resolver for binder_b200.forward.GpuRecursion: filter, upstream table, forward, match and relay on
    the CPU."""

    def __init__(self):
        self.region, self.dcs, self.upstreams = None, [], []

    def set_recursion_filter(self, region, dcs=(), ptr=False):
        self.region, self.dcs = region, list(dcs)

    def set_recursion_upstreams(self, upstreams):
        self.upstreams = list(upstreams)

    def _table(self):
        return Table(self.region, self.dcs, self.upstreams)

    def forward_batch(self, data, off, id_key):
        return forward_batch(self._table(), data, off, id_key)

    def match_upstreams(self, resp, resp_off, src_ip, src_port, q_data, q_off, route, id_key):
        return match_upstreams(self._table(), resp, resp_off, src_ip, src_port, q_data, q_off, route, id_key)

    def relay_batch(self, q_data, q_off, up_data, up_off, tcp=False):
        return relay_oracle.relay_batch(q_data, q_off, up_data, up_off, tcp)
