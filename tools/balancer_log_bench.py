"""What the query log costs the balancer sessions (DESIGN.md section 15): bb_backend_feed of 16,384 INBOUND_UDP frames,
and a bb_tcp_hub flush of 16,384 messages from 64 sessions, with the query log off and on, alternated call by call on
one engine.  Two mixes on the zones tools/log_bench.py uses: config 2's host A lookups and config 3's service mix (50 %
SRV / 50 % A on service names).  Every call is synchronous, so a host clock around it includes the device work.
Reports, as one JSON line:
  per mix and session: median ms per call off and on, the added ms, records per call, records per second of added time
  (and of the whole call), and the run-to-run spread (max - min over median) of each side
  gpu   card name and power limit, read in the same run

    python tools/balancer_log_bench.py [--reps 30] [--warmup 5] [--zone-records 200000] [--out FILE]
"""
import argparse
import json
import os
import struct
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

N = 16384
HUB_SESSIONS = 64


def gpu_info():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else 'unknown'


def summary(ts):
    ts = np.asarray(ts) * 1e3
    med = float(np.median(ts))
    return med, float((ts.max() - ts.min()) / med)


def timed(reps, warmup, calls):
    """calls: {'off': fn, 'on': fn}, each returning a record count; alternated, warm-up first -> {key: [seconds]}"""
    for _ in range(warmup):
        for fn in calls.values():
            fn()
    ts = {k: [] for k in calls}
    recs = {}
    for _ in range(reps):
        for k, fn in calls.items():
            t0 = time.perf_counter()
            recs[k] = fn()
            ts[k].append(time.perf_counter() - t0)
    return ts, recs


def report(ts, recs):
    off, off_spread = summary(ts['off'])
    on, on_spread = summary(ts['on'])
    added = on - off
    r = recs['on']
    return {'ms_off': off, 'ms_on': on, 'added_ms': added, 'records': r,
            'records_per_s_of_added_time': r / (added / 1e3) if added > 0 else None, 'records_per_s_whole_call': r / (on / 1e3),
            'spread_off': off_spread, 'spread_on': on_spread}


def run(name, zone, args):
    from binder_b200 import balancer, synth
    from binder_b200.engine import Engine
    eng = Engine(zone.dns_domain, zone.datacenter, recursion=True, snapshot=zone.jsonl, max_batch=N, ordered=True)
    pkts = synth.batch_service(zone, N, seed=7) if name == 'config3' else synth.batch_host_a(zone, N, seed=7)
    res = {}

    # UDP backend: one feed of N frames (one batch)
    frames = b''.join(struct.pack('<IIII', balancer.INBOUND_UDP, 0x0A000000 + i, 1024 + i % 60000, len(p)) + p
                      for i, p in enumerate(pkts))
    be = {k: balancer.NativeBackend(eng, max_batch=N) for k in ('off', 'on')}
    be['on'].set_query_log(True)

    def feed(k):
        def fn():
            be[k].feed(frames, seed=7)
            return len(be[k].query_log(0).log_len) if k == 'on' else 0
        return fn
    ts, recs = timed(args.reps, args.warmup, {k: feed(k) for k in be})
    res['backend_feed'] = dict(report(ts, recs), answered=be['on'].stats()['answered'], lost=be['on'].stats()['lost'])

    # TCP hub: N messages from 64 sessions, one flush (batches of 4,096: the hub's answer room per batch)
    hub = {k: balancer.NativeTcpHub(eng, max_batch=4096) for k in ('off', 'on')}
    hub['on'].set_query_log(True)
    sids = {}
    for k, h in hub.items():
        sids[k] = [h.open() for _ in range(HUB_SESSIONS)]
        for j, s in enumerate(sids[k]):
            h.feed(s, struct.pack('<III', balancer.INBOUND_TCP, 0x0A010000 + j, 2000 + j))
    streams = [b''.join(struct.pack('>H', len(p)) + p for p in pkts[j::HUB_SESSIONS]) for j in range(HUB_SESSIONS)]
    timings = {'off': [], 'on': []}
    recs = {}
    for rep in range(args.warmup + args.reps):
        for k, h in hub.items():
            for s, st in zip(sids[k], streams):                 # queueing the messages is not timed
                h.feed(s, st)
            t0 = time.perf_counter()
            h.flush(7)
            dt = time.perf_counter() - t0
            recs[k] = len(h.query_log(0).log_len) if k == 'on' else 0
            for s in sids[k]:
                h.consume(s, len(h.output(s)[0]))
            if rep >= args.warmup:
                timings[k].append(dt)
    res['hub_flush'] = dict(report(timings, recs), failed=hub['on'].stats()['failed'], lost=hub['on'].stats()['lost'])
    eng.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=30)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--zone-records', type=int, default=200000)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    from binder_b200 import synth
    res = {'gpu': gpu_info(), 'zone_records': args.zone_records, 'frames_per_call': N}
    res['config2'] = run('config2', synth.gen_zone(args.zone_records), args)
    res['config3'] = run('config3', synth.gen_zone(args.zone_records, service_frac=0.15), args)
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
