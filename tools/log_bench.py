"""Query log throughput (bb_log_batch_device / bb_log_batch, DESIGN.md section 15) over the result sets of config 3
(262,144 service queries: 50 % SRV / 50 % A on service names) and config 2 (65,536 host A lookups), made by the resolve
kernel from seeded batches.  The zone is smaller than the configs' (--zone-records; the records an answer carries, not
the zone's size, decide its log record; DESIGN.md section 15 states the deviation).  Reports, as one JSON line:
  device   records/s and text bytes/s with the result set and the log in HBM (CUDA events, after warm-up)
  e2e      the same through bb_log_batch with pinned host buffers (H2D of the result set, records written to host memory)
  cpu      the Python restatement (tests/query_log_ref.py: dnspython + json.dumps) on a sample, lines/s on one thread
  parity   the device log of the last timed step against bb_log_batch's
  gpu      card name and power limit, read in the same run

    python tools/log_bench.py [--steps 50] [--warmup 10] [--zone-records 200000]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, 'oracle'), os.path.join(ROOT, 'tests')):
    if p not in sys.path:
        sys.path.insert(0, p)


def gpu_info():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else 'unknown'


def pinned(lib, count, dtype):
    nbytes = max(16, count * np.dtype(dtype).itemsize)
    p = lib.bb_host_alloc(nbytes)
    return np.frombuffer((ctypes.c_uint8 * nbytes).from_address(p), dtype=dtype, count=count), p


def run(name, zone, batch, args):
    import torch
    import query_log_ref as L
    from binder_b200 import synth
    from binder_b200._lib import lib
    from binder_b200.engine import Engine
    eng = Engine(zone.dns_domain, zone.datacenter, recursion=True, snapshot=zone.jsonl, max_batch=batch, ordered=True)
    pkts = synth.batch_service(zone, batch, seed=7) if name == 'config3' else synth.batch_host_a(zone, batch, seed=7)
    out, off, lens, st, _ = eng.resolve_batch(*synth.pack_batch(pkts), seed=7)
    off = off[:batch]
    log, log_off, log_len, head_len = eng.log_batch(out, off, lens, st)
    total, recs = len(log), int((log_len > 0).sum())
    dev = torch.device('cuda:0')
    d = dict(out=torch.from_numpy(np.concatenate([out, np.zeros(16, np.uint8)])).to(dev), off=torch.from_numpy(off.view(np.int32)).to(dev),
             ln=torch.from_numpy(lens.view(np.int16)).to(dev), st=torch.from_numpy(st).to(dev),
             log=torch.zeros(total + 64, dtype=torch.uint8, device=dev), lo=torch.zeros(batch + 1, dtype=torch.int32, device=dev),
             ll=torch.zeros(batch, dtype=torch.int32, device=dev), hl=torch.zeros(batch, dtype=torch.int16, device=dev),
             sm=torch.zeros(batch, dtype=torch.int32, device=dev), tot=torch.zeros(4, dtype=torch.int32, device=dev))
    s = torch.cuda.Stream()

    def step():
        eng.log_device(d['out'].data_ptr(), len(out), 0, d['off'].data_ptr(), d['ln'].data_ptr(), d['st'].data_ptr(), batch,
                       d['log'].data_ptr(), total, d['lo'].data_ptr(), d['ll'].data_ptr(), d['hl'].data_ptr(), d['sm'].data_ptr(),
                       d['tot'].data_ptr(), stream=s.cuda_stream)
    for _ in range(args.warmup):
        step()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(s)
    for _ in range(args.steps):
        step()
    e1.record(s)
    torch.cuda.synchronize()
    dev_s = e0.elapsed_time(e1) / 1e3 / args.steps
    got = d['log'].cpu().numpy()[:total]
    parity = bool(np.array_equal(got, log) and np.array_equal(d['lo'].cpu().numpy().view(np.uint32)[:batch], log_off[:batch]))
    # end to end through bb_log_batch with pinned buffers
    bufs = [pinned(lib(), total + 64, np.uint8), pinned(lib(), batch + 1, np.uint32), pinned(lib(), batch, np.uint32),
            pinned(lib(), batch, np.uint16)]
    arrs = tuple(b for b, _ in bufs) + (None,)
    for _ in range(3):
        eng.log_batch(out, off, lens, st, buffers=arrs)
    t0 = time.perf_counter()
    for _ in range(max(1, args.steps // 5)):
        eng.log_batch(out, off, lens, st, buffers=arrs)
    e2e_s = (time.perf_counter() - t0) / max(1, args.steps // 5)
    for _, p in bufs:
        lib().bb_host_free(p)
    # the restatement on one thread, on a sample
    k = min(batch, 4000)
    t0 = time.perf_counter()
    L.log_set(out, off[:k], lens[:k], st[:k], zone.dns_domain)
    cpu_lps = k / (time.perf_counter() - t0)
    eng.close()
    return {'records': recs, 'text_bytes': total, 'device': {'records_per_s': recs / dev_s, 'text_bytes_per_s': total / dev_s,
            'ms_per_call': dev_s * 1e3}, 'e2e': {'records_per_s': recs / e2e_s, 'ms_per_call': e2e_s * 1e3},
            'cpu_restatement_lines_per_s': cpu_lps, 'parity': parity}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=50)
    ap.add_argument('--warmup', type=int, default=10)
    ap.add_argument('--zone-records', type=int, default=200000)
    args = ap.parse_args()
    from binder_b200 import synth
    res = {'gpu': gpu_info(), 'zone_records': args.zone_records}
    res['config3'] = run('config3', synth.gen_zone(args.zone_records, service_frac=0.15), 262144, args)
    res['config2'] = run('config2', synth.gen_zone(args.zone_records), 65536, args)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
