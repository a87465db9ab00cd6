"""Query log on the GPU (DESIGN.md section 15): Engine.log_batch and the device-resident form byte for byte against the
restatement (tests/query_log_ref.py) on the engine's own result sets (resolve in both packings, UDP and TCP, and relays),
hand-written and malformed responses; batch sizes up to 1,048,576 (there against the device source on the CPU,
tests/native/emu_log.cpp, and a seeded sample against the restatement); pinned and pageable results; tiles whose
responses exceed the staging buffer or are scattered; a resolve -> log chain that reads the resolve totals on the device;
capacity; several streams at once; argument errors."""
import ctypes
import random

import numpy as np
import pytest

import fuzzgen
import query_log_ref as L
import relaygen as G
from binder_b200 import synth
from binder_b200._lib import BinderError, lib
from binder_b200.engine import Engine
from test_query_log import emu_exe, emu_log, hand_responses, malformed_responses, pack_set, relay_set

pytestmark = pytest.mark.gpu
_ENG = {}


def fuzz_engine(ordered, max_batch=1 << 20):
    key = ('fuzz', ordered, max_batch)
    if key not in _ENG:
        snap, info = fuzzgen.gen_zone(3)
        _ENG[key] = (Engine(info['dns_domain'], 'dc1', recursion=True, snapshot=snap, max_batch=max_batch, ordered=ordered), info)
    return _ENG[key]


def relay_engine(ordered):
    key = ('relay', ordered)
    if key not in _ENG:
        _ENG[key] = Engine('dc2.example.com', 'dc1', recursion=True, max_batch=1 << 20, ordered=ordered)
    return _ENG[key]


def records(res):
    log, log_off, log_len, head_len, summ = res
    out = []
    for i in range(len(log_len)):
        rec = bytes(log[log_off[i]:log_off[i] + log_len[i]])
        out.append((rec[:head_len[i]], rec[head_len[i]:], int(summ[i])))
    return out


def check(eng, rs, dom, want=None, **kw):
    res = eng.log_batch(*rs, summary=True, **kw)
    got = records(res)
    want = L.log_set(*rs, dom) if want is None else want
    assert len(got) == len(want)
    for i, (g, w) in enumerate(zip(got, want)):
        assert g == w, (i, g, w)
    if eng.ordered:                                  # query order: the records are packed back to back
        assert np.array_equal(res[1][1:len(got)], (res[1][:len(got)] + res[2]).astype(np.uint32)[:-1])
    return got


def fuzz_result_set(eng, info, seed, tcp, n=3000):
    pkts = fuzzgen.gen_queries(seed, info, n) + fuzzgen.malformed_packets()
    out, off, lens, st, _ = eng.resolve_batch(*synth.pack_batch(pkts), seed=seed, tcp=tcp)
    return out, off, lens, st


@pytest.mark.parametrize('ordered', [False, True])
@pytest.mark.parametrize('tcp', [False, True])
def test_gpu_log_resolve_and_relay_sets(ordered, tcp):
    eng, info = fuzz_engine(ordered)
    rs = fuzz_result_set(eng, info, 20 + tcp, tcp)
    got = check(eng, rs, info['dns_domain'])
    assert sum(1 for h, _, _ in got if h) > 1000 and any(s == 1 for s in rs[3])
    re = relay_engine(ordered)
    rel = relay_set(30 + tcp, tcp)
    pairs_rs = re.relay_batch(*G.pack_pairs(G.gen_relays(32 + tcp, 2000)), tcp=tcp)
    check(re, rel, 'dc2.example.com')
    check(re, pairs_rs, 'dc2.example.com')


@pytest.mark.parametrize('ordered', [False, True])
def test_gpu_log_hand_written_and_malformed(ordered):
    eng = relay_engine(ordered)
    resps = hand_responses() + list(malformed_responses().values())
    rs = pack_set(resps)
    got = check(eng, rs, 'dc2.example.com')
    assert [s for _, _, s in got[-len(malformed_responses()):]] == [L.BAD] * len(malformed_responses())
    out, off, lens, st = rs
    off = off.copy()
    off[0] = len(out) + 1                            # outside the response bytes
    got = check(eng, (out, off, lens, st), 'dc2.example.com')
    assert got[0] == (b'', b'', L.BAD)


def tiled_set(n, seed=5, scatter=False):
    """n responses over one base buffer: in order (each tile contiguous) or at random offsets (scattered tiles)."""
    eng, info = fuzz_engine(False)
    out, off, lens, st = fuzz_result_set(eng, info, seed, False, 1500)
    base = [bytes(out[off[i]:off[i] + lens[i]]) for i in range(len(st))] + hand_responses()
    bst = list(st) + [0] * len(hand_responses())
    rng = random.Random(seed)
    idx = [rng.randrange(len(base)) for _ in range(n)] if scatter else [i % len(base) for i in range(n)]
    if scatter:
        b_out, b_off, b_len, _ = pack_set(base)
        return (b_out, b_off[idx] if n else b_off[:1], b_len[idx], np.asarray(bst, np.uint8)[idx]), info['dns_domain']
    return pack_set([base[i] for i in idx], [bst[i] for i in idx]), info['dns_domain']


@pytest.mark.parametrize('n', [0, 1, 127, 128, 129, 65536, 1048576])
def test_gpu_log_batch_sizes(n, tmp_path_factory, tmp_path):
    for scatter in (False, True):
        rs, dom = tiled_set(n, scatter=scatter)
        if n <= 65536:
            want = L.log_set(*rs, dom)
        else:
            want = emu_log(emu_exe(tmp_path_factory), rs, dom, tmp_path)
            sample = sorted(random.Random(n + scatter).sample(range(n), 20000))
            out, off, lens, st = rs
            assert [want[i] for i in sample] == L.log_set(out, off[sample], lens[sample], st[sample], dom)
        for ordered in (False, True):
            check(fuzz_engine(ordered)[0], rs, dom, want=want)


def pinned(count, dtype):
    nbytes = max(16, count * np.dtype(dtype).itemsize)
    p = lib().bb_host_alloc(nbytes)
    assert p
    buf = (ctypes.c_uint8 * nbytes).from_address(p)
    return np.frombuffer(buf, dtype=dtype, count=count), p


@pytest.mark.parametrize('ordered', [False, True])
@pytest.mark.parametrize('with_summary', [False, True])
def test_gpu_log_pinned_results(ordered, with_summary):
    eng, info = fuzz_engine(ordered)
    rs = fuzz_result_set(eng, info, 40, True)
    n = len(rs[3])
    want = L.log_set(*rs, info['dns_domain'])
    total = sum(len(h) + len(b) for h, b, _ in want)
    bufs = [pinned(total + 64, np.uint8), pinned(n + 1, np.uint32), pinned(n, np.uint32), pinned(n, np.uint16), pinned(n, np.uint32)]
    try:
        arrs = [b for b, _ in bufs]
        if not with_summary:
            arrs[4] = None
        res = eng.log_batch(*rs, summary=with_summary, buffers=tuple(arrs))
        got = records(res if with_summary else res + (np.array([w[2] for w in want], np.uint32),))
        assert got == want
    finally:
        for _, p in bufs:
            lib().bb_host_free(p)


@pytest.mark.parametrize('ordered', [False, True])
def test_gpu_log_tiles_past_staging(ordered):
    """TCP responses of many A records (tens of KB each) and long relayed replies: tiles far past the 32 KB staging."""
    eng = relay_engine(ordered)
    rng = random.Random(8)
    pairs = [G.relay_case(rng, 'expand') for _ in range(40)] + [G.relay_case(rng, 'many') for _ in range(300)]
    rs = eng.relay_batch(*G.pack_pairs(pairs), tcp=True)
    got = check(eng, rs, 'dc2.example.com')
    assert max(len(h) + len(b) for h, b, _ in got) > 65535


def test_gpu_log_capacity_and_args():
    eng, info = fuzz_engine(False)
    rs = fuzz_result_set(eng, info, 50, False, 500)
    n = len(rs[3])
    want = L.log_set(*rs, info['dns_domain'])
    total = sum(len(h) + len(b) for h, b, _ in want)
    for cap, ok in ((total - 1, False), (total, True)):
        bufs = (np.zeros(cap, np.uint8), np.zeros(n + 1, np.uint32), np.zeros(n, np.uint32), np.zeros(n, np.uint16), np.zeros(n, np.uint32))
        if ok:
            assert records(eng.log_batch(*rs, summary=True, buffers=bufs)) == want
        else:
            with pytest.raises(BinderError) as ei:
                eng.log_batch(*rs, summary=True, buffers=bufs)
            assert ei.value.code == -5
    small, _ = fuzz_engine(False, max_batch=256)
    big = fuzz_result_set(eng, info, 51, False, 300)
    with pytest.raises(BinderError) as ei:
        small.log_batch(*big)
    assert ei.value.code == -1


def _dev(torch, a, dtype=None):
    t = torch.from_numpy(np.ascontiguousarray(a) if dtype is None else np.ascontiguousarray(a).view(dtype))
    return t.to('cuda:0')


def test_gpu_log_device_streams_and_chain():
    import torch
    dev = torch.device('cuda:0')
    eng, info = fuzz_engine(True)
    dom = info['dns_domain']
    batches = []
    for k, size in enumerate((1, 129, 3000, 700, 128)):
        pkts = (fuzzgen.gen_queries(60 + k, info, size) + fuzzgen.malformed_packets())[:size]
        data, off = synth.pack_batch(pkts)
        n = len(pkts)
        rs = eng.resolve_batch(data, off, seed=k)[:4]
        want = L.log_set(*rs, dom)
        total = sum(len(h) + len(b) for h, b, _ in want)
        t = dict(pk=_dev(torch, np.concatenate([data, np.zeros(16, np.uint8)])), po=_dev(torch, off, np.int32),
                 out=torch.zeros(n * 1232 + 64, dtype=torch.uint8, device=dev), oo=torch.zeros(n + 1, dtype=torch.int32, device=dev),
                 ol=torch.zeros(n, dtype=torch.int16, device=dev), st=torch.zeros(n, dtype=torch.uint8, device=dev),
                 miss=torch.zeros(n, dtype=torch.int32, device=dev), rt=torch.zeros(8, dtype=torch.int32, device=dev),
                 log=torch.zeros(total + 64, dtype=torch.uint8, device=dev), lo=torch.zeros(n + 1, dtype=torch.int32, device=dev),
                 ll=torch.zeros(n, dtype=torch.int32, device=dev), hl=torch.zeros(n, dtype=torch.int16, device=dev),
                 sm=torch.zeros(n, dtype=torch.int32, device=dev), tot=torch.zeros(4, dtype=torch.int32, device=dev))
        batches.append((n, t, want, total, torch.cuda.Stream()))

    def log_args(n, t, cap):
        return (t['out'].data_ptr(), n * 1232, t['rt'].data_ptr(), t['oo'].data_ptr(), t['ol'].data_ptr(), t['st'].data_ptr(), n,
                t['log'].data_ptr(), cap, t['lo'].data_ptr(), t['ll'].data_ptr(), t['hl'].data_ptr(), t['sm'].data_ptr(), t['tot'].data_ptr())

    def fetch(t, n, tot):
        return records((t['log'].cpu().numpy()[:tot[0]], t['lo'].cpu().numpy().view(np.uint32), t['ll'].cpu().numpy().view(np.uint32),
                        t['hl'].cpu().numpy().view(np.uint16), t['sm'].cpu().numpy().view(np.uint32)))

    epochs = []
    for rep in range(3):                 # resolve -> log on each stream, all enqueued before any synchronisation
        for k, (n, t, want, total, s) in enumerate(batches):
            eng.resolve_device(t['pk'].data_ptr(), t['po'].data_ptr(), n, k, 0, t['out'].data_ptr(), n * 1232, t['oo'].data_ptr(),
                               t['ol'].data_ptr(), t['st'].data_ptr(), t['miss'].data_ptr(), t['rt'].data_ptr(), stream=s.cuda_stream)
            eng.log_device(*log_args(n, t, total), stream=s.cuda_stream)
            epochs.append(lib().bb_engine_launch_epoch(eng._h))
    torch.cuda.synchronize()
    for i, (n, t, want, total, s) in enumerate(batches):
        tot = t['tot'].cpu().numpy().view(np.uint32)
        ep = epochs[10 + i]
        assert tot[0] == total and tot[1] == sum(1 for h, _, _ in want if h) and tot[2] != ep and tot[3] == ep
        assert fetch(t, n, tot) == want
    # overflow (one byte short), then an exact launch on the same stream
    n, t, want, total, s = batches[2]
    eng.log_device(*log_args(n, t, total - 1), stream=s.cuda_stream)
    ep = lib().bb_engine_launch_epoch(eng._h)
    torch.cuda.synchronize()
    tot = t['tot'].cpu().numpy().view(np.uint32)
    assert tot[2] == ep and tot[3] == ep
    eng.log_device(*log_args(n, t, total), stream=s.cuda_stream)
    ep2 = lib().bb_engine_launch_epoch(eng._h)
    torch.cuda.synchronize()
    tot = t['tot'].cpu().numpy().view(np.uint32)
    assert tot[2] == ep and tot[3] == ep2 and tot[0] == total and fetch(t, n, tot) == want
    # BB_ERR_ARG: misaligned response or log buffer, n > max_batch
    a = list(log_args(n, t, total))
    for k in (0, 7):
        b = list(a)
        b[k] += 1
        with pytest.raises(BinderError) as ei:
            eng.log_device(*b, stream=s.cuda_stream)
        assert ei.value.code == -1
    small, _ = fuzz_engine(True, max_batch=256)
    b = list(a)
    b[6] = 257
    with pytest.raises(BinderError) as ei:
        small.log_device(*b)
    assert ei.value.code == -1
    torch.cuda.synchronize()
