"""Recursion relay on the GPU (DESIGN.md section 13): Engine.relay_batch bit-exact against the relay oracle on the relay
corpora, in both packings, over UDP and TCP; batch-size edges up to 1,048,576 relays; pinned (zero-copy) and pageable
results; tiles whose bytes exceed the staging buffers; the device-resident form on several streams."""
import ctypes
import random

import numpy as np
import pytest

import relay_oracle
import relaygen as G
from binder_b200 import synth
from binder_b200._lib import BinderError, lib
from binder_b200.engine import Engine, repack
from test_relay import corpus

pytestmark = pytest.mark.gpu
_ENG = {}


def engine(ordered, max_batch=1 << 20):
    key = (ordered, max_batch)
    if key not in _ENG:
        _ENG[key] = Engine('example.com', 'dc1', recursion=True, max_batch=max_batch, ordered=ordered)
    return _ENG[key]


def check(got, want, ordered):
    out, ooff, olen, st = got
    wout, woff, wlen, wst = want
    n = len(wst)
    assert np.array_equal(st, wst) and np.array_equal(olen, wlen)
    if ordered:
        assert np.array_equal(ooff[:n + 1], woff)
    packed, poff = repack(out, ooff[:n + 1], olen)
    assert np.array_equal(poff, woff) and np.array_equal(packed, wout)


def oracle(pairs_or_packed, tcp=False):
    packed = pairs_or_packed if isinstance(pairs_or_packed, tuple) else G.pack_pairs(pairs_or_packed)
    return relay_oracle.relay_batch(*packed, tcp=tcp, nthreads=8)


@pytest.mark.parametrize('ordered', [False, True])
@pytest.mark.parametrize('tcp', [False, True])
def test_gpu_relay_matches_oracle(ordered, tcp):
    pairs = corpus(41 + tcp, 3000)
    packed = G.pack_pairs(pairs)
    check(engine(ordered).relay_batch(*packed, tcp=tcp), oracle(packed, tcp), ordered)


def _tiled(n, seed=5):
    base = [p for p in corpus(seed, 600) if len(p[1]) < 2000]
    return [base[i % len(base)] for i in range(n)]


@pytest.mark.parametrize('n', [0, 1, 127, 128, 129, 65536, 1048576])
def test_gpu_relay_batch_sizes(n):
    pairs = _tiled(n)
    packed = G.pack_pairs(pairs) if n else (np.zeros(16, np.uint8), np.zeros(1, np.uint32), np.zeros(16, np.uint8), np.zeros(1, np.uint32))
    want = oracle(packed)
    for ordered in (False, True):
        check(engine(ordered).relay_batch(*packed), want, ordered)


def pinned(count, dtype):
    nbytes = max(16, count * np.dtype(dtype).itemsize)
    p = lib().bb_host_alloc(nbytes)
    assert p
    buf = (ctypes.c_uint8 * nbytes).from_address(p)
    return np.frombuffer(buf, dtype=dtype, count=count), p


@pytest.mark.parametrize('ordered', [False, True])
@pytest.mark.parametrize('tcp', [False, True])
def test_gpu_relay_pinned_results(ordered, tcp):
    pairs = corpus(51, 2000) + [G.relay_case(random.Random(i), 'expand') for i in range(40)]
    packed = G.pack_pairs(pairs)
    n = len(pairs)
    want = oracle(packed, tcp)
    bufs = [pinned(len(want[0]) + 64, np.uint8), pinned(n + 1, np.uint32), pinned(n, np.uint16), pinned(n, np.uint8)]
    try:
        got = engine(ordered).relay_batch(*packed, tcp=tcp, out=tuple(b for b, _ in bufs))
        check(got, want, ordered)
    finally:
        for _, p in bufs:
            lib().bb_host_free(p)


@pytest.mark.parametrize('ordered', [False, True])
def test_gpu_relay_tiles_past_staging(ordered):
    """Tiles whose query bytes (> 8 KB: trailing bytes after each question) or upstream bytes (> 24 KB) are not staged."""
    rng = random.Random(8)
    pairs = [G.relay_case(rng, 'expand') for _ in range(300)]
    pairs += [(q + bytes(rng.randrange(256) for _ in range(100)), u) for q, u in G.gen_relays(9, 600)]
    pairs += G.gen_relays(10, 300)
    for tcp in (False, True):
        packed = G.pack_pairs(pairs)
        check(engine(ordered).relay_batch(*packed, tcp=tcp), oracle(packed, tcp), ordered)


def test_gpu_relay_capacity_and_args():
    pairs = corpus(61, 500)
    packed = G.pack_pairs(pairs)
    want = oracle(packed)
    total = len(want[0])
    e = engine(False)
    for cap, ok in ((total, True), (total - 1, False)):
        out = (np.zeros(cap, np.uint8), np.zeros(len(pairs) + 1, np.uint32), np.zeros(len(pairs), np.uint16), np.zeros(len(pairs), np.uint8))
        if ok:
            check(e.relay_batch(*packed, out=out), want, False)
        else:
            with pytest.raises(BinderError) as ei:
                e.relay_batch(*packed, out=out)
            assert ei.value.code == -5
    q_data, q_off, up_data, up_off = packed
    bad = up_off.copy()
    bad[3] = bad[4] + 1                             # offsets that decrease
    with pytest.raises(BinderError) as ei:
        e.relay_batch(q_data, q_off, up_data, bad)
    assert ei.value.code == -1
    small = engine(False, max_batch=256)
    with pytest.raises(BinderError) as ei:
        small.relay_batch(*G.pack_pairs(corpus(62, 300)))
    assert ei.value.code == -1
    norec = Engine('example.com', 'dc1', recursion=False, max_batch=1024)
    with pytest.raises(BinderError) as ei:
        norec.relay_batch(*G.pack_pairs(pairs[:10]))
    assert ei.value.code == -1


def test_gpu_relay_device_resident_streams():
    import torch
    dev = torch.device('cuda:0')
    e = engine(True)
    batches = []
    for k, size in enumerate((1, 129, 3000, 700, 128)):
        pairs = corpus(70 + k, size)[:size]
        q_data, q_off, up_data, up_off = packed = G.pack_pairs(pairs)
        want = oracle(packed)
        n = len(pairs)
        t = dict(q=torch.from_numpy(np.concatenate([q_data, np.zeros(16, np.uint8)])).to(dev),
                 qo=torch.from_numpy(q_off.view(np.int32)).to(dev),
                 u=torch.from_numpy(np.concatenate([up_data, np.zeros(16, np.uint8)])).to(dev),
                 uo=torch.from_numpy(up_off.view(np.int32)).to(dev),
                 out=torch.zeros(len(want[0]) + 64, dtype=torch.uint8, device=dev), off=torch.zeros(n + 1, dtype=torch.int32, device=dev),
                 ln=torch.zeros(n, dtype=torch.int16, device=dev), st=torch.zeros(n, dtype=torch.uint8, device=dev),
                 tot=torch.zeros(4, dtype=torch.int32, device=dev))
        batches.append((n, t, want, torch.cuda.Stream()))
    epochs = []
    for rep in range(3):                            # three launches per stream, all enqueued before any synchronisation
        for n, t, want, s in batches:
            e.relay_device(t['q'].data_ptr(), t['qo'].data_ptr(), t['u'].data_ptr(), t['uo'].data_ptr(), n, t['out'].data_ptr(),
                           len(want[0]), t['off'].data_ptr(), t['ln'].data_ptr(), t['st'].data_ptr(), t['tot'].data_ptr(),
                           stream=s.cuda_stream)
            epochs.append(lib().bb_engine_launch_epoch(e._h))
    torch.cuda.synchronize()
    for i, (n, t, want, s) in enumerate(batches):
        tot = t['tot'].cpu().numpy().view(np.uint32)
        assert tot[0] == len(want[0]) and tot[1] == 0 and tot[2] != epochs[10 + i] and tot[3] == epochs[10 + i]
        got = (t['out'].cpu().numpy()[:tot[0]], t['off'].cpu().numpy().view(np.uint32), t['ln'].cpu().numpy().view(np.uint16),
               t['st'].cpu().numpy())
        check(got, want, True)
    # overflow (one byte short), then an exact launch on the same stream
    n, t, want, s = batches[2]
    args = lambda cap: (t['q'].data_ptr(), t['qo'].data_ptr(), t['u'].data_ptr(), t['uo'].data_ptr(), n, t['out'].data_ptr(), cap,   # noqa: E731
                        t['off'].data_ptr(), t['ln'].data_ptr(), t['st'].data_ptr(), t['tot'].data_ptr())
    e.relay_device(*args(len(want[0]) - 1), stream=s.cuda_stream)
    ep = lib().bb_engine_launch_epoch(e._h)
    torch.cuda.synchronize()
    tot = t['tot'].cpu().numpy().view(np.uint32)
    assert tot[2] == ep and tot[3] == ep
    e.relay_device(*args(len(want[0])), stream=s.cuda_stream)
    ep2 = lib().bb_engine_launch_epoch(e._h)
    torch.cuda.synchronize()
    tot = t['tot'].cpu().numpy().view(np.uint32)
    assert tot[2] == ep and tot[3] == ep2 and tot[0] == len(want[0])
    check((t['out'].cpu().numpy()[:tot[0]], t['off'].cpu().numpy().view(np.uint32), t['ln'].cpu().numpy().view(np.uint16),
           t['st'].cpu().numpy()), want, True)
    # BB_ERR_ARG: misaligned buffers, n > max_batch, a 17th stream
    a = list(args(len(want[0])))
    for k in (0, 2, 5):
        b = list(a)
        b[k] += 1
        with pytest.raises(BinderError) as ei:
            e.relay_device(*b, stream=s.cuda_stream)
        assert ei.value.code == -1
    small = engine(True, max_batch=256)
    b = list(a)
    b[4] = 257
    with pytest.raises(BinderError) as ei:
        small.relay_device(*b)
    assert ei.value.code == -1
    extra = [torch.cuda.Stream() for _ in range(16)]
    with pytest.raises(BinderError) as ei:
        for x in extra:
            e.relay_device(*a, stream=x.cuda_stream)
    assert ei.value.code == -1
    torch.cuda.synchronize()
