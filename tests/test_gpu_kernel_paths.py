"""The routes through the resolve kernel that the parity tests' single host call does not take, each checked against
oracle/liboracle.so with the checks of assert_same:

  A. zero-copy results: every output buffer pinned (bb_host_alloc), so the kernel writes straight into host memory
     (big tiles through the device bounce buffer, emit rounds flushed with 16-byte stores), four slots in flight,
     capacity edges, a slot switching buffer sets, and whether zero-copy actually engaged (no device-to-host copies);
  B. device-resident launches on several streams at once: per-stream look-back scratch, self-cleaning between
     launches, the totals contract (bytes, misses, overflow marker, done marker), argument errors, and the automatic
     variant switch driven by the feedback ring;
  C. batches of several waves of tiles (262,144 and 1,048,576 queries; the ordered look-back then walks more than one
     window of predecessors), and a batch that fills max_batch and max_batch_bytes exactly;
  D. input edges: a query index that wraps inside the batch, a seed with only its high half set, a batch that does not
     start at byte 0, zero-length packets, packets around the 65,535-byte limit.
"""
import ctypes
import json
import os

import numpy as np
import pytest

import fuzzgen
import helpers as H
from binder_b200 import synth
from binder_b200._lib import lib, check
from test_gpu_parity import compare, staging_case, MODES
from test_host_emulation import job_zone, padded_queries, size_zone
from test_tcp import big_zone, big_zone_batch

pytestmark = pytest.mark.gpu

ERR_ARG, ERR_CAPACITY, BATCH_TCP = -1, -5, 1
PROFILES = ['small', 'service']


# ---- zones and batches, built once ----------------------------------------------------------------------------------
def _staging_case():
    """Tiles larger than the shared-memory staging take the direct path (through the bounce buffer when results are
    pinned)."""
    snap, pkts = staging_case()
    return 'foo.com', snap, False, pkts


def _fuzz_case():
    snap, info = fuzzgen.gen_zone(7, n_top=40)
    pkts = fuzzgen.gen_queries(7, info, n=3000) + fuzzgen.malformed_packets() + fuzzgen.tolerated_packets()
    return info['dns_domain'], snap, True, pkts


def _jobs_case():
    """Big tiles of service answers (the batch of test_copy_jobs_edges, EDNS sizes mixed): many emit rounds, more copy
    jobs than the list holds, SRV runs cut short by truncation, upper-case names in between."""
    pkts = []
    for i in range(3000):
        s = (i * 7) % 24
        name = 'svc%02d.foo.com' % s
        if i % 11 == 0:
            name = name.upper()[:5] + name[5:]
        edns = (0, 1200, 700)[i % 5 % 3]
        pkts.append(synth.make_query(name, 'A', i, edns=edns) if i % 3 == 2 else
                    synth.make_query('_http._tcp.' + name, 'SRV', i, edns=edns))
    return 'foo.com', job_zone(), False, pkts


def _big_case():
    return 'foo.com', big_zone(), False, big_zone_batch()


CASES = {'fuzz': _fuzz_case, 'jobs': _jobs_case, 'staging': _staging_case, 'big': _big_case}


class World(object):
    """Per case: the zone, its batch, an oracle, and engines (one per packing) created on first use."""

    def __init__(self):
        self.cases, self.engines, self.oracle_results = {}, {}, {}

    def case(self, name):
        if name not in self.cases:
            dom, snap, rec, pkts = CASES[name]()
            data, off = synth.pack_batch(pkts)
            self.cases[name] = dict(dom=dom, snap=snap, rec=rec, data=data, off=off,
                                    orc=H.make_impl('oracle', dom, snap, recursion=rec))
        return self.cases[name]

    def engine(self, name, ordered, **kw):
        key = (name, ordered) + tuple(sorted(kw.items()))
        if key not in self.engines:
            c = self.case(name)
            self.engines[key] = H.make_impl('gpu', c['dom'], c['snap'], recursion=c['rec'], ordered=ordered, **kw)
        return self.engines[key]

    def oracle(self, name, data, off, seed, qidx_base=0, tcp=False):
        key = (name, id(data), seed, qidx_base, tcp)
        if key not in self.oracle_results:
            self.oracle_results[key] = (data, self.case(name)['orc'].resolve_batch(
                data, off, seed=seed, qidx_base=qidx_base, tcp=tcp, nthreads=os.cpu_count()))
        return self.oracle_results[key][1]


@pytest.fixture(scope='module')
def world():
    w = World()
    yield w
    for e in w.engines.values():
        e.close()


# ---- output buffers and the submit/wait calls ---------------------------------------------------------------------
class Outputs(object):
    """out, out_off, out_len, status and miss_idx of one batch, each pinned (bb_host_alloc) or pageable (numpy).
    Pinned memory is released only by release(), so no two live sets ever share an address."""

    def __init__(self, n, cap, pinned=('out', 'out_off', 'out_len', 'status', 'miss')):
        self.ptrs = []
        sizes = dict(out=(cap, np.uint8), out_off=(n + 1, np.uint32), out_len=(n, np.uint16), status=(n, np.uint8),
                     miss=(n, np.uint32))
        for k, (count, dt) in sizes.items():
            count = max(count, 1)
            if k in pinned:
                nb = count * np.dtype(dt).itemsize
                p = lib().bb_host_alloc(nb)
                assert p, 'bb_host_alloc(%d) failed' % nb
                self.ptrs.append(p)
                a = np.ctypeslib.as_array((ctypes.c_uint8 * nb).from_address(p)).view(dt)
            else:
                a = np.empty(count, dtype=dt)
            setattr(self, k, a)
        self.reset()

    def reset(self):
        """Stale bytes everywhere: whatever the next call does not write stays visibly wrong."""
        for k in ('out', 'out_off', 'out_len', 'status', 'miss'):
            getattr(self, k).view(np.uint8)[:] = 0xA7
        self.n_miss = ctypes.c_uint32(0xFFFFFFFF)

    def release(self):
        for p in self.ptrs:
            lib().bb_host_free(p)
        self.ptrs = []


@pytest.fixture
def outputs():
    made = []

    def make(*a, **kw):
        made.append(Outputs(*a, **kw))
        return made[-1]
    yield make
    for o in made:
        o.release()


def submit(eng, slot, data, off, o, seed, qidx_base=0, tcp=False, out_cap=None):
    return lib().bb_resolve_submit_ex(eng._h, slot, data.ctypes.data, off.ctypes.data, len(off) - 1, seed, qidx_base,
                                      o.out.ctypes.data, o.out.size if out_cap is None else out_cap, o.out_off.ctypes.data,
                                      o.out_len.ctypes.data, o.status.ctypes.data, o.miss.ctypes.data,
                                      ctypes.byref(o.n_miss), BATCH_TCP if tcp else 0)


def results(o, n):
    return (o.out[:o.out_off[n]].copy(), o.out_off[:n + 1].copy(), o.out_len[:n].copy(), o.status[:n].copy(),
            o.miss[:o.n_miss.value].copy())


def run_slot(eng, slot, data, off, o, seed, **kw):
    check(submit(eng, slot, data, off, o, seed, **kw))
    check(lib().bb_resolve_wait(eng._h, slot))
    return results(o, len(off) - 1)


def cuda_trace(fn, tmp_path):
    """Run fn under torch.profiler (CUDA activity) -> (names of resolve kernels launched, device-to-host copies);
    None when the profiler recorded no CUDA activity at all."""
    import torch
    from torch.profiler import profile, ProfilerActivity
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    path = str(tmp_path / ('trace_%d.json' % len(os.listdir(str(tmp_path)))))
    prof.export_chrome_trace(path)
    with open(path) as f:
        ev = json.load(f).get('traceEvents', [])
    kernels = [e.get('name', '') for e in ev if e.get('cat') == 'kernel']
    copies = [e.get('name', '') for e in ev if e.get('cat') == 'gpu_memcpy']
    if not kernels and not copies:
        return None
    return [k for k in kernels if 'resolve_kernel' in k], sum('DtoH' in c for c in copies)


# ---- A. pinned (zero-copy) results ---------------------------------------------------------------------------------
@pytest.mark.parametrize('tcp', [False, True], ids=['udp', 'tcp'])
@pytest.mark.parametrize('profile', PROFILES)
@pytest.mark.parametrize('ordered', MODES)
def test_pinned_results_match_oracle(world, outputs, ordered, profile, tcp):
    for k, name in enumerate(CASES):
        c = world.case(name)
        data, off = c['data'], c['off']
        n = len(off) - 1
        o_res = world.oracle(name, data, off, seed=31 + k, qidx_base=1000 * k, tcp=tcp)
        eng = world.engine(name, ordered)
        eng.set_kernel_profile(profile)
        o = outputs(n, len(o_res[0]) + 4096)
        res = run_slot(eng, k % 4, data, off, o, 31 + k, qidx_base=1000 * k, tcp=tcp)
        compare(res, o_res, data, off, ordered)


@pytest.mark.parametrize('ordered', MODES)
def test_pinned_four_slots_in_flight(outputs, ordered):
    """All four slots in flight at once, two rounds, distinct batches and qidx_bases, each checked after its wait."""
    z = synth.gen_zone(50000, service_frac=0.15)
    eng = H.make_impl('gpu', z.dns_domain, z.jsonl, recursion=True, ordered=ordered)
    orc = H.make_impl('oracle', z.dns_domain, z.jsonl, recursion=True)
    try:
        for rnd in range(2):
            jobs = []
            for s in range(4):
                i = rnd * 4 + s
                pk = synth.batch_mixed(z, 3000 + 977 * i, seed=200 + i, miss_frac=0.2) + synth.batch_service(z, 1500 * (i % 3), seed=300 + i)
                data, off = synth.pack_batch(pk)
                o = outputs(len(off) - 1, (len(off) - 1) * 600)
                check(submit(eng, s, data, off, o, 55 + i, qidx_base=7919 * i))
                jobs.append((data, off, o, i))
            for s, (data, off, o, i) in enumerate(jobs):
                check(lib().bb_resolve_wait(eng._h, s))
                compare(results(o, len(off) - 1), orc.resolve_batch(data, off, seed=55 + i, qidx_base=7919 * i), data, off, ordered)
    finally:
        eng.close()


@pytest.mark.parametrize('profile', PROFILES)
@pytest.mark.parametrize('ordered', MODES)
def test_pinned_capacity_edges(world, outputs, ordered, profile):
    """out_cap equal to the batch's bytes is enough, one byte less is BB_ERR_CAPACITY, and the slot then resolves the
    next batch exactly."""
    c = world.case('jobs')
    data, off = c['data'], c['off']
    n = len(off) - 1
    eng = world.engine('jobs', ordered)
    eng.set_kernel_profile(profile)
    o_res = world.oracle('jobs', data, off, seed=4)
    total = len(o_res[0])
    o = outputs(n, total)
    compare(run_slot(eng, 2, data, off, o, 4, out_cap=total), o_res, data, off, ordered)
    check(submit(eng, 2, data, off, o, 4, out_cap=total - 1))
    assert lib().bb_resolve_wait(eng._h, 2) == ERR_CAPACITY
    o2 = outputs(n, total + 64)
    compare(run_slot(eng, 2, data, off, o2, 5), world.oracle('jobs', data, off, seed=5), data, off, ordered)


@pytest.mark.parametrize('ordered', MODES)
def test_pinned_slot_switches_buffer_sets(world, outputs, ordered):
    """One slot: pinned -> pageable -> pinned again -> only `out` pinned; every result exact."""
    for name in ('jobs', 'big'):
        c = world.case(name)
        data, off = c['data'], c['off']
        n = len(off) - 1
        eng = world.engine(name, ordered)
        eng.set_kernel_profile('auto')
        tcp = name == 'big'
        cap = len(world.oracle(name, data, off, seed=60, tcp=tcp)[0]) + 4096
        pinned = outputs(n, cap)
        sets = [pinned, outputs(n, cap, pinned=()), pinned, outputs(n, cap, pinned=('out',))]
        for k, o in enumerate(sets):
            o.reset()
            res = run_slot(eng, 1, data, off, o, 60 + k, tcp=tcp)
            compare(res, world.oracle(name, data, off, seed=60 + k, tcp=tcp), data, off, ordered)


def test_zero_copy_engages(world, outputs, tmp_path):
    """Pinned buffers: no device-to-host copy at all (the kernel wrote the results); pageable buffers: copies.  Also on
    a slot whose first submit with those pinned buffers was an empty batch."""
    c = world.case('jobs')
    data, off = c['data'], c['off']
    n = len(off) - 1
    eng = H.make_impl('gpu', c['dom'], c['snap'], recursion=c['rec'])
    try:
        o_res = world.oracle('jobs', data, off, seed=8)
        runs = {}
        pinned, pageable, late = outputs(n, n * 1232), outputs(n, n * 1232, pinned=()), outputs(n, n * 1232)
        empty_data, empty_off = np.zeros(16, np.uint8), np.zeros(1, np.uint32)

        def run(key, slot, o):
            runs[key] = run_slot(eng, slot, data, off, o, 8)
        run('warm', 0, pinned)
        tr = {'pinned': cuda_trace(lambda: run('pinned', 0, pinned), tmp_path),
              'pageable': cuda_trace(lambda: run('pageable', 0, pageable), tmp_path)}
        # slot 3's first submit with `late` is an empty batch: the next one with the same buffers must still be zero-copy
        empty = run_slot(eng, 3, empty_data, empty_off, late, 8)
        assert empty[1][0] == 0 and late.n_miss.value == 0
        tr['after_empty'] = cuda_trace(lambda: run('after_empty', 3, late), tmp_path)
        for key, res in runs.items():
            compare(res, o_res, data, off, False)
        if any(t is None for t in tr.values()):
            pytest.skip('the profiler recorded no CUDA activity: results checked, zero-copy not observable')
        for key, (kernels, d2h) in tr.items():
            assert kernels, (key, 'no resolve kernel in the trace')
        assert tr['pinned'][1] == 0, tr
        assert tr['pageable'][1] > 0, tr
        assert tr['after_empty'][1] == 0, ('an empty first submit turned zero-copy off for these buffers', tr)
    finally:
        eng.close()


# ---- B. device-resident launches ------------------------------------------------------------------------------------
class DevBatch(object):
    """A batch and its output buffers in device memory (torch); the byte array is padded to a multiple of 16."""

    def __init__(self, data, off, out_cap=None):
        import torch
        dev = torch.device('cuda:0')
        self.data, self.off, self.n = data, off, len(off) - 1
        assert data.size % 16 == 0 and data.size >= off[-1]
        n1 = max(self.n, 1)
        self.d_pk = torch.from_numpy(np.concatenate([data, np.zeros(16, np.uint8)])).to(dev)
        self.d_off = torch.from_numpy(off.view(np.int32)).to(dev)
        self.cap = out_cap if out_cap is not None else max(self.n * 600, 4096)
        self.d_out = torch.empty(self.cap + 16, dtype=torch.uint8, device=dev)
        self.d_oo = torch.full((self.n + 1,), -1, dtype=torch.int32, device=dev)
        self.d_ol = torch.full((n1,), -1, dtype=torch.int16, device=dev)
        self.d_st = torch.full((n1,), 0xA7, dtype=torch.uint8, device=dev)
        self.d_ms = torch.full((n1,), -1, dtype=torch.int32, device=dev)
        self.d_tot = torch.full((4,), -1, dtype=torch.int32, device=dev)

    def launch(self, eng, seed, qidx_base=0, stream=0, out_cap=None, n=None, d_pkts=None, d_out=None):
        """-> (return code, bb_engine_launch_epoch() right after the call)"""
        rc = lib().bb_resolve_batch_device(eng._h, self.d_pk.data_ptr() if d_pkts is None else d_pkts, self.d_off.data_ptr(),
                                           self.n if n is None else n, seed, qidx_base,
                                           self.d_out.data_ptr() if d_out is None else d_out, self.cap if out_cap is None else out_cap,
                                           self.d_oo.data_ptr(), self.d_ol.data_ptr(), self.d_st.data_ptr(), self.d_ms.data_ptr(),
                                           self.d_tot.data_ptr(), stream)
        return rc, int(lib().bb_engine_launch_epoch(eng._h))

    def totals(self):
        return self.d_tot.cpu().numpy().view(np.uint32)

    def results(self):
        tot = self.totals()
        n = self.n
        return (self.d_out[:int(tot[0])].cpu().numpy(), self.d_oo.cpu().numpy().view(np.uint32),
                self.d_ol[:n].cpu().numpy().view(np.uint16), self.d_st[:n].cpu().numpy(),
                self.d_ms[:int(tot[1])].cpu().numpy().view(np.uint32))

    def check(self, orc, seed, epoch, ordered, qidx_base=0, **kw):
        """Exact against the oracle, and the totals: bytes, misses, no overflow marker, the done marker = epoch."""
        o_res = orc.resolve_batch(self.data, self.off, seed=seed, qidx_base=qidx_base, **kw)
        tot = self.totals()
        assert tot[0] == len(o_res[0]) and tot[1] == len(o_res[4]), (tot, len(o_res[0]), len(o_res[4]))
        assert tot[3] == epoch and tot[2] != epoch, (tot, epoch)
        compare(self.results(), o_res, self.data, self.off, ordered)


@pytest.fixture(scope='module')
def svc_zone():
    z = synth.gen_zone(50000, service_frac=0.15)
    return z, H.make_impl('oracle', z.dns_domain, z.jsonl, recursion=True)


WORK = ['config2', 'config3', 'config4', 'config5']


def gen(z, n, seed, workload):
    _, _, mix, miss_frac, _ = synth.WORKLOADS[workload]
    data, off, _ = synth.gen_batch(z, n, seed, mix, miss_frac)
    return data, off


@pytest.mark.parametrize('ordered', MODES)
def test_device_launches_on_five_streams(svc_zone, ordered):
    """Four torch streams and the default stream, three launches each, all enqueued before anything synchronises."""
    import torch
    z, orc = svc_zone
    eng = H.make_impl('gpu', z.dns_domain, z.jsonl, recursion=True, ordered=ordered)
    try:
        streams = [torch.cuda.Stream() for _ in range(4)]
        ptrs = [s.cuda_stream for s in streams] + [0]
        sizes = [1, 129, 5000, 65536]
        batches = []
        for k in range(3):
            for j in range(5):
                i = k * 5 + j
                batches.append((DevBatch(*gen(z, sizes[i % 4], 500 + i, WORK[(i + k) % 4])), ptrs[j], i))
        torch.cuda.synchronize()
        epochs = []
        for b, st, i in batches:
            rc, ep = b.launch(eng, 1000 + i, qidx_base=i << 20, stream=st)
            check(rc)
            epochs.append(ep)
        assert len(set(epochs)) == len(epochs)
        torch.cuda.synchronize()
        for (b, st, i), ep in zip(batches, epochs):
            b.check(orc, 1000 + i, ep, ordered, qidx_base=i << 20)
    finally:
        eng.close()


@pytest.mark.parametrize('ordered', MODES)
def test_device_overflow_then_exact(svc_zone, ordered):
    """Too small an out_cap sets the overflow marker to the launch's epoch; the next launch on the stream is exact."""
    import torch
    z, orc = svc_zone
    eng = H.make_impl('gpu', z.dns_domain, z.jsonl, recursion=True, ordered=ordered)
    try:
        b = DevBatch(*gen(z, 20000, 77, 'config3'))
        st = torch.cuda.Stream()
        rc, ep1 = b.launch(eng, 3, stream=st.cuda_stream, out_cap=4096)
        check(rc)
        st.synchronize()
        assert b.totals()[2] == ep1 and b.totals()[3] == ep1
        rc, ep2 = b.launch(eng, 3, stream=st.cuda_stream)
        check(rc)
        st.synchronize()
        b.check(orc, 3, ep2, ordered)
    finally:
        eng.close()


@pytest.mark.parametrize('ordered', MODES)
def test_device_empty_batch_sets_done_marker(svc_zone, ordered):
    import torch
    z, orc = svc_zone
    eng = H.make_impl('gpu', z.dns_domain, z.jsonl, recursion=True, ordered=ordered)
    try:
        b = DevBatch(np.zeros(16, np.uint8), np.zeros(1, np.uint32))
        rc, ep = b.launch(eng, 1)
        check(rc)
        torch.cuda.synchronize()
        tot = b.totals()
        assert b.d_oo.cpu().numpy()[0] == 0
        assert tot[0] == 0 and tot[1] == 0 and tot[3] == ep, (tot, ep)
        # and the launch after it is exact
        b2 = DevBatch(*gen(z, 3000, 9, 'config4'))
        rc, ep = b2.launch(eng, 2)
        check(rc)
        torch.cuda.synchronize()
        b2.check(orc, 2, ep, ordered)
    finally:
        eng.close()


def test_device_argument_errors(svc_zone):
    """Misaligned d_pkts or d_out, n > max_batch and a 17th distinct stream are BB_ERR_ARG; the first 16 streams keep
    working."""
    import torch
    z, orc = svc_zone
    eng = H.make_impl('gpu', z.dns_domain, z.jsonl, recursion=True, ordered=True, max_batch=4096)
    try:
        b = DevBatch(*gen(z, 300, 1, 'config4'))
        for k in (1, 4, 8):
            assert b.launch(eng, 1, d_pkts=b.d_pk.data_ptr() + k)[0] == ERR_ARG
            assert b.launch(eng, 1, d_out=b.d_out.data_ptr() + k)[0] == ERR_ARG
        assert b.launch(eng, 1, n=4097)[0] == ERR_ARG
        streams = [torch.cuda.Stream() for _ in range(17)]
        outs = [DevBatch(b.data, b.off) for _ in range(16)]
        for s, o in zip(streams, outs):
            check(o.launch(eng, 1, stream=s.cuda_stream)[0])
        assert b.launch(eng, 1, stream=streams[16].cuda_stream)[0] == ERR_ARG
        torch.cuda.synchronize()
        for rnd in range(2):
            eps = []
            for s, o in zip(streams, outs):
                rc, ep = o.launch(eng, 10 + rnd, stream=s.cuda_stream)
                check(rc)
                eps.append(ep)
            torch.cuda.synchronize()
            for o, ep in zip(outs, eps):
                o.check(orc, 10 + rnd, ep, True)
    finally:
        eng.close()


@pytest.mark.parametrize('ordered', MODES)
def test_device_auto_profile_follows_feedback(svc_zone, ordered, tmp_path):
    """Profile 'auto' on one stream: batches of 64-byte answers (config 2) and of service answers (config 3) in turn.
    The feedback ring makes the variant follow the previous batch, so both variants run both shapes; every launch is
    exact."""
    import torch
    z, orc = svc_zone
    eng = H.make_impl('gpu', z.dns_domain, z.jsonl, recursion=True, ordered=ordered)
    try:
        eng.set_kernel_profile('auto')
        st = torch.cuda.Stream()
        shapes = ['config2', 'config2', 'config3', 'config3'] * 2
        batches = [DevBatch(*gen(z, 20000, 40 + i, w)) for i, w in enumerate(shapes)]
        torch.cuda.synchronize()
        done = []

        def go():
            for i, b in enumerate(batches):
                rc, ep = b.launch(eng, 70 + i, stream=st.cuda_stream)
                check(rc)
                st.synchronize()                     # the next launch sees this one's feedback
                done.append(ep)
        tr = cuda_trace(go, tmp_path)
        for i, (b, ep) in enumerate(zip(batches, done)):
            b.check(orc, 70 + i, ep, ordered)
        mean = [b.totals()[0] / b.n for b in batches]
        assert max(mean[0], mean[1]) < 96 <= min(mean[2], mean[3]), mean
        if tr is not None:
            assert len(set(tr[0])) == 2, sorted(set(tr[0]))     # both variants ran
    finally:
        eng.close()


# ---- C. batches of several waves -----------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def wave_world():
    """The config-3 zone of test_gpu_parity (300,000 records, 15 % services), engines for 2^20 queries per batch."""
    z = synth.gen_zone(300000, service_frac=0.15)
    orc = H.make_impl('oracle', z.dns_domain, z.jsonl, recursion=True)
    engines = {o: H.make_impl('gpu', z.dns_domain, z.jsonl, recursion=True, ordered=o, max_batch=1 << 20) for o in (False, True)}
    cache = {}

    def batch(name):
        if name not in cache:
            if name == 'config3':
                data, off = gen(z, 262144, 3, 'config3')
            elif name == 'config4':
                _, _, mix, _, _ = synth.WORKLOADS['config4']
                data, off, _ = synth.gen_batch(z, 1 << 20, 4, mix, 0.2)
            else:                                     # 'full': 2^20 packets of 64 bytes = max_batch_bytes exactly
                data, off = gen(z, 1 << 20, 5, 'config4')
                lens = np.diff(off.astype(np.int64))
                assert lens.max() <= 64
                rows = np.full((1 << 20, 64), 0x5A, dtype=np.uint8)          # trailing bytes after each question
                start = off[:-1].astype(np.int64)
                for k in range(64):
                    m = lens > k
                    rows[m, k] = data[start[m] + k]
                data, off = rows.reshape(-1), (np.arange((1 << 20) + 1, dtype=np.int64) * 64).astype(np.uint32)
            cache[name] = (data, off, orc.resolve_batch(data, off, seed=0x5EED, nthreads=os.cpu_count()))
        return cache[name]
    yield engines, batch
    for e in engines.values():
        e.close()


@pytest.mark.parametrize('ordered', MODES)
@pytest.mark.parametrize('name', ['config3', 'config4', 'full'])
def test_multi_wave_host_path(wave_world, name, ordered):
    engines, batch = wave_world
    data, off, o_res = batch(name)
    eng = engines[ordered]
    if name == 'full':
        assert len(off) - 1 == lib().bb_engine_max_batch(eng._h) and off[-1] == lib().bb_engine_max_batch_bytes(eng._h)
    compare(eng.resolve_batch(data, off, seed=0x5EED), o_res, data, off, ordered)
    if name == 'config4':
        assert len(o_res[4]) > 100000                 # recursion misses over the whole batch


def test_multi_wave_device_path_ordered(wave_world):
    import torch
    engines, batch = wave_world
    data, off, o_res = batch('config4')
    b = DevBatch(data, off, out_cap=len(o_res[0]) + 4096)
    rc, ep = b.launch(engines[True], 0x5EED)
    check(rc)
    torch.cuda.synchronize()
    tot = b.totals()
    assert tot[0] == len(o_res[0]) and tot[1] == len(o_res[4]) and tot[3] == ep and tot[2] != ep
    compare(b.results(), o_res, data, off, True)


# ---- D. input edges -------------------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def edge_world():
    z = synth.gen_zone(3000, service_frac=0.3)
    orc = H.make_impl('oracle', z.dns_domain, z.jsonl, recursion=True)
    engines = {o: H.make_impl('gpu', z.dns_domain, z.jsonl, recursion=True, ordered=o) for o in (False, True)}
    yield z, orc, engines
    for e in engines.values():
        e.close()


def _check(eng, orc, data, off, **kw):
    o_res = orc.resolve_batch(data, off, **kw)
    res = eng.resolve_batch(data, off, **kw)
    return compare(res, o_res, data, off, eng.ordered)


@pytest.mark.parametrize('ordered', MODES)
def test_query_index_wraps_inside_batch(edge_world, ordered):
    """qidx_base = 2^32 - 200: the index wraps to 0 at query 200 and keeps keying the shuffle from there."""
    z, orc, engines = edge_world
    pk = synth.batch_service(z, 1000, seed=12, srv_frac=0.6)
    data, off = synth.pack_batch(pk)
    packed, poff = _check(engines[ordered], orc, data, off, seed=21, qidx_base=2 ** 32 - 200)[:2]
    d2, o2 = synth.pack_batch(pk[200:])
    p2 = _check(engines[ordered], orc, d2, o2, seed=21, qidx_base=0)[0]
    assert np.array_equal(packed[poff[200]:], p2)            # the wrapped indices are 0, 1, ... again


@pytest.mark.parametrize('ordered', MODES)
def test_seed_high_half_only(edge_world, ordered):
    z, orc, engines = edge_world
    data, off = synth.pack_batch(synth.batch_service(z, 1000, seed=13, srv_frac=0.6))
    hi = _check(engines[ordered], orc, data, off, seed=0xC0FFEE11 << 32)[0]
    lo = _check(engines[ordered], orc, data, off, seed=0)[0]
    assert not np.array_equal(hi, lo)                        # the high half of the seed changes the shuffle


@pytest.mark.parametrize('ordered', MODES)
def test_batch_not_starting_at_byte_zero(edge_world, ordered):
    z, orc, engines = edge_world
    data, off = synth.pack_batch(synth.batch_mixed(z, 1000, seed=14, miss_frac=0.2))
    d5 = np.concatenate([np.full(5, 0xEE, np.uint8), data, np.zeros(11, np.uint8)])
    _check(engines[ordered], orc, d5, off + np.uint32(5), seed=22)


@pytest.mark.parametrize('ordered', MODES)
def test_zero_length_packets(edge_world, ordered):
    """Empty packets in the middle of a tile, and a whole tile (queries 256..383) of them."""
    z, orc, engines = edge_world
    pk = synth.batch_mixed(z, 600, seed=15)
    pk = pk[:40] + [b''] * 3 + pk[40:100] + [b''] + pk[100:]
    pk = pk[:256] + [b''] * 128 + pk[256:]
    data, off = synth.pack_batch(pk)
    g = _check(engines[ordered], orc, data, off, seed=23)
    assert (g[3][256:384] == 2).all() and (g[3][40:43] == 2).all()


@pytest.mark.parametrize('tcp', [False, True], ids=['udp', 'tcp'])
@pytest.mark.parametrize('ordered', MODES)
def test_packets_around_the_length_limit(ordered, tcp):
    """Packets of 65,534 / 65,535 bytes are queries (trailing bytes ignored), 65,536 and 70,000 bytes are dropped."""
    snap = size_zone()
    eng = H.make_impl('gpu', 'foo.com', snap, ordered=ordered)
    orc = H.make_impl('oracle', 'foo.com', snap)
    try:
        data, off = synth.pack_batch(padded_queries([65534, 65535, 65536, 70000, 65535, 70000]))
        g = _check(eng, orc, data, off, seed=5, tcp=tcp)
        assert list(g[3][0::2]) == [0, 0, 2, 2, 0, 2] and (g[3][1::2] == 0).all()
    finally:
        eng.close()
