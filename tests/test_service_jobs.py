"""The copy-job count that size_service() takes while it sizes a service answer, against a TaskCount walk of
plan_service() over the same answer, for every job-mode answer (tests/native/emu_service_jobs.cpp: the device source
on the CPU).  Also: no query walks its service's children more often than the kernel did before the count moved into
the sizing walk."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest

import fuzzgen
import helpers as H
from binder_b200 import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NSTAT = 11


def jobs_lib(tmp):
    """The driver built with -DBB_EMU_WALKS (walk steps counted); shared with tools/walk_counts.py."""
    cxx = shutil.which('g++')
    if not cxx:
        pytest.skip('no g++')
    so = os.path.join(str(tmp), 'libbbjobs.so')
    srcs = [os.path.join(ROOT, 'tests', 'native', 'emu_service_jobs.cpp'), os.path.join(ROOT, 'binder_b200', 'csrc', 'zone_build.cpp')]
    subprocess.check_call([cxx, '-std=c++17', '-O1', '-fPIC', '-shared', '-Wno-unknown-pragmas', '-DBB_EMU_WALKS',
                           '-I', os.path.join(ROOT, 'include'), '-I', os.path.join(ROOT, 'binder_b200', 'csrc'), '-o', so] + srcs)
    L = ctypes.CDLL(so)
    L.bb_zone_build.restype = ctypes.c_void_p
    L.bb_zone_build.argtypes = [ctypes.c_char_p, ctypes.c_size_t, ctypes.c_char_p, ctypes.POINTER(ctypes.c_int)]
    L.bb_zone_free.argtypes = [ctypes.c_void_p]
    L.bb_emu_service_jobs.argtypes = [ctypes.c_void_p, ctypes.c_char_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_uint32, ctypes.c_uint64,
                                      ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
    return L


class Zone(object):
    def __init__(self, L, dns_domain, snap):
        self.L, self.dom = L, dns_domain.encode()
        err = ctypes.c_int(0)
        self.z = L.bb_zone_build(snap, len(snap), self.dom, ctypes.byref(err))
        assert self.z, err.value

    def run(self, pkts, seed, tcp=False):
        """-> (stats[NSTAT], steps now, steps before, is_srv) over the packed batch"""
        data, off = synth.pack_batch(pkts) if isinstance(pkts, list) else pkts
        data = np.ascontiguousarray(data, dtype=np.uint8); off = np.ascontiguousarray(off, dtype=np.uint32)
        n = len(off) - 1
        st = np.zeros(NSTAT, dtype=np.uint64)
        now, before, srv = np.zeros(n, np.uint32), np.zeros(n, np.uint32), np.zeros(n, np.uint8)
        rc = self.L.bb_emu_service_jobs(self.z, self.dom, data.ctypes.data, off.ctypes.data, n, seed, int(tcp), st.ctypes.data,
                                        now.ctypes.data, before.ctypes.data, srv.ctypes.data)
        assert rc == 0, rc
        assert st[9] == 0, 'job count differs from the TaskCount walk (first at query %d)' % int(st[10])
        assert (now <= before).all(), 'a query walks its children more often than before'
        return st, now, before, srv

    def close(self):
        self.L.bb_zone_free(self.z)


@pytest.fixture(scope='module')
def L(tmp_path_factory):
    return jobs_lib(tmp_path_factory.mktemp('jobs'))


# a dnsDomain so long that 16 A answers no longer fit 512 bytes behind the question
LONG_DOMAIN = '.'.join(['a' * 60, 'b' * 60, 'c' * 60, 'd' * 50, 'com'])


def sixteen_zone(dns_domain='foo.com'):
    """Services of 16 children (and one of 17, never job mode): multi-port children, long and short child names, null
    addresses, and malformed children (no load_balancer object) in some of them."""
    top = '/' + '/'.join(reversed(dns_domain.split('.')))
    ent = [(top, None)]
    for s in range(14):
        nk = 17 if s == 13 else 16
        ent.append((top + '/w%02d' % s, {'type': 'service', 'service': {'srvce': '_http', 'proto': '_tcp', 'port': 80, 'ttl': 60}}))
        for k in range(nk):
            if s % 4 == 1 and k == (s * 5) % 16:
                rec = {'type': 'load_balancer', 'x': 1}
            elif s % 4 == 2 and k % 7 == 3:
                rec = {'type': 'load_balancer', 'load_balancer': {'address': None}}
            elif (s + k) % 3 == 0:
                rec = {'type': 'rr_host', 'rr_host': {'address': '10.%d.%d.1' % (s, k), 'ports': [9000 + i for i in range(1 + (s + k) % 4)]}}
            else:
                rec = {'type': 'load_balancer', 'load_balancer': {'address': '10.%d.%d.2' % (s, k)}}
            ent.append((top + '/w%02d/%s%d' % (s, 'a-rather-long-backend-name-' if k % 4 == 0 else 'b', k), rec))
    return H.snapshot(ent)


def service_queries(names, n, edns_choices, dns_domain='foo.com'):
    pk = []
    for i in range(n):
        name = names[(i * 7) % len(names)] + '.' + dns_domain
        edns = edns_choices[i % len(edns_choices)]
        pk.append(synth.make_query(name if i % 3 == 2 else '_http._tcp.' + name, 'A' if i % 3 == 2 else 'SRV', i & 0xFFFF, edns=edns))
    return pk


def test_job_count_sixteen_children_and_malformed(L):
    z = Zone(L, 'foo.com', sixteen_zone())
    pk = service_queries(['w%02d' % s for s in range(14)], 1400, [None, 1200, 700, 560])
    tot = np.zeros(NSTAT, dtype=np.uint64)
    for seed in (1, 2, 3):
        st, now, before, _ = z.run(pk, seed)
        tot += st
        assert (now < before).any()
    st, _, _, _ = z.run(pk, 4, tcp=True)
    tot += st
    z.close()
    z = Zone(L, LONG_DOMAIN, sixteen_zone(LONG_DOMAIN))
    tot += z.run(service_queries(['w%02d' % s for s in range(14)], 600, [None, 600], LONG_DOMAIN), 9)[0]
    z.close()
    checked, tr_srv, tr_a, masked, add_cut, edns, bad_whole, bad_tr, sixteen = [int(x) for x in tot[:9]]
    assert checked > 3000 and tr_srv and tr_a and masked and add_cut and edns and sixteen > 1000, list(tot)
    assert bad_whole and bad_tr, list(tot)            # a malformed child before the truncation cut and after it


def test_job_count_copy_job_zone(L):
    from test_host_emulation import job_zone
    z = Zone(L, 'foo.com', job_zone())
    pk = service_queries(['svc%02d' % s for s in range(24)], 1000, [None, 1200, 700])
    tot = np.zeros(NSTAT, dtype=np.uint64)
    for seed in (5, 6):
        tot += z.run(pk, seed)[0]
    z.close()
    assert tot[0] > 1000 and tot[1] and tot[3] and tot[4] and tot[5], list(tot)


@pytest.mark.parametrize('seed', range(8))
def test_job_count_fuzz_zones(L, seed):
    snap, info = fuzzgen.gen_zone(seed, n_top=40)
    z = Zone(L, info['dns_domain'], snap)
    pkts = fuzzgen.gen_queries(seed, info, n=3000)
    z.run(pkts, seed * 7 + 1)
    z.run(pkts, seed + 2, tcp=True)
    z.close()


def test_job_count_config3_shape(L):
    desc, service_frac, mix, miss_frac, recursion = synth.WORKLOADS['config3']
    zone = synth.gen_zone(30000, service_frac=service_frac)
    z = Zone(L, zone.dns_domain, zone.jsonl)
    data, off, meta = synth.gen_batch(zone, 8192, 5, mix, miss_frac)
    st, now, before, srv = z.run((data, off), 11)
    z.close()
    assert st[0] > 6000 and st[1] > 0, list(st)
    # truncated SRV answers walk their children less often than before; the rest as often
    assert now[srv == 1].sum() < before[srv == 1].sum()
