"""Child-walk steps per 32-query warp of the service variant, now and as the kernel walked before size_service()
counted the copy jobs (tests/native/emu_service_jobs.cpp: the device source on the CPU, -DBB_EMU_WALKS).  A warp runs
its lanes' walks in lockstep, so its cost is the longest lane's; warps are formed the way the kernel forms them (per
128-query tile, the SRV queries after the others).  Deterministic: a seeded batch of the workload on a synthetic zone.

    python tools/walk_counts.py [--workload config3] [--zone-records 1000000] [--batch 262144] [--seed 3]
"""
import argparse
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'tests'), os.path.join(ROOT, 'oracle')]
from binder_b200 import synth  # noqa: E402
from test_service_jobs import jobs_lib, Zone  # noqa: E402


def warp_max(steps, is_srv, tile=128, warp=32):
    """max over the lanes of each warp, SRV queries grouped after the others inside each tile -> (per-warp max, warp is SRV)"""
    out, kind = [], []
    for q0 in range(0, len(steps), tile):
        s, v = steps[q0:q0 + tile], is_srv[q0:q0 + tile]
        order = np.concatenate([np.nonzero(v == 0)[0], np.nonzero(v == 1)[0]])
        s, v = s[order], v[order]
        for w0 in range(0, len(s), warp):
            out.append(int(s[w0:w0 + warp].max()))
            kind.append(bool(v[w0:w0 + warp].any()))
    return np.array(out), np.array(kind)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--workload', default='config3', choices=sorted(synth.WORKLOADS))
    ap.add_argument('--zone-records', type=int, default=1000000)
    ap.add_argument('--batch', type=int, default=262144)
    ap.add_argument('--seed', type=int, default=3)
    a = ap.parse_args()
    desc, service_frac, mix, miss_frac, recursion = synth.WORKLOADS[a.workload]
    zone = synth.gen_zone(a.zone_records, service_frac=service_frac)
    data, off, meta = synth.gen_batch(zone, a.batch, a.seed, mix, miss_frac)
    with tempfile.TemporaryDirectory() as tmp:
        z = Zone(jobs_lib(tmp), zone.dns_domain, zone.jsonl)
        st, now, before, srv = z.run((data, off), a.seed)
        z.close()
    print('%s, %d records, %d queries, seed %d: %d job-mode service answers, %d of them truncated SRV'
          % (a.workload, a.zone_records, a.batch, a.seed, int(st[0]), int(st[1])))
    wb, kind = warp_max(before, srv)
    wn, _ = warp_max(now, srv)
    print('%-26s %10s %10s %8s' % ('child-walk steps', 'before', 'now', 'ratio'))
    for label, m in (('per warp (max lane), all', np.ones_like(kind)), ('per warp, SRV warps', kind), ('per warp, other warps', ~kind)):
        if m.any():
            b, n = wb[m].mean(), wn[m].mean()
            print('%-26s %10.2f %10.2f %8.3f' % (label, b, n, n / b if b else float('nan')))
    print('%-26s %10d %10d %8.3f' % ('all lanes, total', int(before.sum()), int(now.sum()), now.sum() / max(before.sum(), 1)))


if __name__ == '__main__':
    main()
