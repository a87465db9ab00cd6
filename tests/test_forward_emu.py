"""The forward and match device source (binder_b200/csrc/forward_device.cuh, through tests/native/emu_forward.cpp) on
the CPU: bit-exact against the forward oracle on the miss corpora of every filter shape and on generated and
hand-written response sets, and clean under AddressSanitizer and UndefinedBehaviorSanitizer on malformed datagrams."""
import os
import random
import shutil
import struct
import subprocess

import numpy as np
import pytest

import forward_oracle as O
import forward_ref as R
import forwardgen as G
from binder_b200 import synth
from binder_b200.engine import ip_u32
from test_recursion_filter import FILTERS

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_EXE = {}


def emu_exe(tmp_factory, sanitize=False):
    if sanitize not in _EXE:
        cxx = shutil.which('g++')
        if not cxx:
            pytest.skip('no g++')
        exe = str(tmp_factory.mktemp('emu_forward') / 'emu_forward')
        san = ['-g', '-fsanitize=address,undefined', '-fno-sanitize-recover=undefined', '-fno-omit-frame-pointer'] if sanitize else []
        b = subprocess.run([cxx, '-std=c++17', '-O1', '-Wno-unknown-pragmas'] + san + ['-I', os.path.join(ROOT, 'include'),
                            '-I', os.path.join(ROOT, 'binder_b200', 'csrc'), '-o', exe, os.path.join(ROOT, 'tests', 'native', 'emu_forward.cpp')],
                           capture_output=True, text=True)
        if sanitize and b.returncode != 0 and 'sanitize' in b.stderr:
            pytest.skip('toolchain without sanitizer runtimes')
        assert b.returncode == 0, b.stderr[-3000:]
        _EXE[sanitize] = exe
    return _EXE[sanitize]


def emu(exe, region, dcs, ups, pkts, items, key, tmp_path):
    """-> (route per miss, upstream query per miss, winner response index per miss or None)."""
    data, off = synth.pack_batch(pkts)
    rd, ro, rip, rport = G.pack(items)
    n, m = len(pkts), len(items)
    buf = struct.pack('<I', len(dcs)) + b''.join(struct.pack('<I', len(d)) + d.encode('latin-1') for d in dcs)
    buf += struct.pack('<I', len(region)) + region.encode('latin-1') + struct.pack('<I', len(ups))
    buf += np.array([ip_u32(a) for a, _, _ in ups], np.uint32).tobytes() + np.array([p for _, p, _ in ups], np.uint16).tobytes()
    buf += np.array([d for _, _, d in ups], np.uint8).tobytes() + struct.pack('<QI', key, n) + off.tobytes() + data[:off[n]].tobytes()
    buf += struct.pack('<I', m) + ro.tobytes() + rip.tobytes() + rport.tobytes() + rd[:ro[m]].tobytes()
    src, dst = str(tmp_path / 'in.bin'), str(tmp_path / 'out.bin')
    open(src, 'wb').write(buf)
    p = subprocess.run([exe, src, dst], capture_output=True, text=True, timeout=600,
                       env=dict(os.environ, ASAN_OPTIONS='detect_leaks=0:abort_on_error=1'))
    assert p.returncode == 0 and p.stdout.startswith('OK') and 'runtime error' not in p.stderr, p.stderr[-3000:]
    raw = open(dst, 'rb').read()
    route = list(raw[:n])
    uq_off = np.frombuffer(raw[n:n + 4 * (n + 1)], np.uint32)
    uq = raw[n + 4 * (n + 1):n + 4 * (n + 1) + int(uq_off[n])]
    win = np.frombuffer(raw[n + 4 * (n + 1) + int(uq_off[n]):], np.uint32)
    return route, [uq[uq_off[j]:uq_off[j + 1]] for j in range(n)], [None if w == 0xFFFFFFFF else int(w) for w in win]


def check(exe, fi, items_of, tmp_path, key):
    region, dcs, _ = FILTERS[fi]
    ups = G.upstream_table(dcs, random.Random(fi))
    pkts = G.misses(fi)
    tb = O.Table(region, dcs, ups)
    data, off = synth.pack_batch(pkts)
    uq, uq_off, order, _, route = O.forward_batch(tb, data, off, key)
    routes, msgs = R.forward(region, dcs, ups, pkts, key)
    for name, items in items_of(ups, pkts, routes, msgs).items():
        e_route, e_msgs, e_win = emu(exe, region, dcs, ups, pkts, items, key, tmp_path)
        assert e_route == route.tolist()
        by_j = {int(j): bytes(uq[uq_off[k]:uq_off[k + 1]]) for k, j in enumerate(order)}
        assert e_msgs == [by_j[j] for j in range(len(pkts))]
        up, up_off = O.match_upstreams(tb, *G.pack(items), data, off, route, key)
        assert [items[w][0] if w is not None else b'' for w in e_win] == \
            [bytes(up[up_off[j]:up_off[j + 1]]) for j in range(len(pkts))], name


def response_sets(key):
    def sets(ups, pkts, routes, msgs):
        out = {'generated': G.responses(ups, routes, msgs, random.Random(5), key)}
        if any(m and r < R.R_PTR for r, m in zip(routes, msgs)):
            out.update(G.hand_written(ups, pkts, routes, msgs, key)[1])
        return out
    return sets


@pytest.mark.parametrize('fi', range(len(FILTERS)))
def test_emulated_forward_is_bit_exact(fi, tmp_path_factory, tmp_path):
    key = 0x9E37 * (fi + 1) << 24
    check(emu_exe(tmp_path_factory), fi, response_sets(key), tmp_path, key)


def mutate(rng, data):
    """Random damage to a datagram: truncation, flipped bytes, a bogus QDCOUNT or label length."""
    b = bytearray(data)
    for _ in range(rng.randint(1, 4)):
        x = rng.random()
        if x < 0.3 and b:
            del b[rng.randrange(len(b)):]
        elif x < 0.6 and b:
            b[rng.randrange(len(b))] = rng.randrange(256)
        elif x < 0.8 and len(b) > 12:
            b[12] = rng.choice([0, 63, 64, 0xC0, 0xFF])
        elif len(b) > 6:
            b[4:6] = struct.pack('>H', rng.choice([0, 1, 2, 0xFFFF]))
    return bytes(b)


def test_emulated_match_is_sanitizer_clean(tmp_path_factory, tmp_path):
    """The hand-written set and a few thousand damaged responses (sources right, IDs valid) under ASan/UBSan."""
    key = 0x1234567890ABCDEF

    def sets(ups, pkts, routes, msgs):
        rng = random.Random(17)
        good = G.responses(ups, routes, msgs, rng, key)
        out = {'damaged': [(mutate(rng, d), s) for d, s in good for _ in range(3)]}
        out.update(G.hand_written(ups, pkts, routes, msgs, key)[1])
        return out
    check(emu_exe(tmp_path_factory, sanitize=True), 0, sets, tmp_path, key)
