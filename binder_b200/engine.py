"""Python face of the C ABI: Zone (the ZKCache read side) and Engine (the query handler).

Mirrors the objects binder wires together in main.js:154-217:
    zkCache = new core.ZKCache({domain})          -> Zone(snapshot, domain)
    server  = core.createServer({zkCache, dnsDomain, datacenterName, recursion})
                                                  -> Engine(dns_domain, datacenter, recursion)
Every call goes through libbinder_b200.so; nothing here computes a DNS answer.
"""
import ctypes

import numpy as np

from . import _lib
from ._lib import check, lib

ANSWERED, MISS_RECURSE, DROPPED = 0, 1, 2


def repack(out, out_off, out_len):
    """Responses re-packed in query order (what ordered_output=1 produces directly)."""
    n = len(out_len)
    lens = out_len.astype(np.int64)
    total = int(lens.sum())
    if total == 0:
        return np.zeros(0, dtype=np.uint8), np.zeros(n + 1, dtype=np.uint32)
    starts = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(lens, out=starts[1:])
    idx = np.repeat(out_off[:n].astype(np.int64) - starts[:n], lens) + np.arange(total)
    return out[idx], starts.astype(np.uint32)


class Zone(object):
    """bb_zone: flattened image of the mirrored ZooKeeper subtree (lib/zk.js ZKCache)."""

    def __init__(self, snapshot_jsonl, dns_domain, nranks=1, rank=0):
        if isinstance(snapshot_jsonl, str):
            snapshot_jsonl = snapshot_jsonl.encode('utf-8')
        err = ctypes.c_int(0)
        self._h = lib().bb_zone_build_shard(snapshot_jsonl, len(snapshot_jsonl), dns_domain.encode(), nranks, rank,
                                            ctypes.byref(err))
        if not self._h:
            raise _lib.BinderError(err.value)

    def stat(self):
        L = lib()
        keys = ('nodes', 'forward_keys', 'reverse_keys', 'slots', 'image_bytes', 'arena_bytes')
        return {k: int(L.bb_zone_stat(self._h, i)) for i, k in enumerate(keys)}

    def apply(self, delta_jsonl):
        """Watch events (dataChanged / childrenChanged, lib/zk.js:120-208) as JSON lines; see bb_zone_apply."""
        if isinstance(delta_jsonl, str):
            delta_jsonl = delta_jsonl.encode('utf-8')
        check(lib().bb_zone_apply(self._h, delta_jsonl, len(delta_jsonl)))

    def pending(self):
        """(slots changed since the device last saw the table, table laid out again?)"""
        return int(lib().bb_zone_stat(self._h, 6)), bool(lib().bb_zone_stat(self._h, 7))

    def probe(self, key, reverse=False):
        """Diagnostics: (kind, ttl, val, payload bytes) the image holds for a key, or None."""
        if isinstance(key, str):
            key = key.encode('latin-1')
        kind, ttl, val, rl = ctypes.c_uint8(0), ctypes.c_uint32(0), ctypes.c_uint32(0), ctypes.c_uint32(0)
        buf = ctypes.create_string_buffer(1 << 16)
        if not lib().bb_zone_probe(self._h, 1 if reverse else 0, key, len(key), ctypes.byref(kind), ctypes.byref(ttl),
                                   ctypes.byref(val), buf, len(buf), ctypes.byref(rl)):
            return None
        return kind.value, ttl.value, val.value, buf.raw[:rl.value]

    def close(self):
        if getattr(self, '_h', None):
            lib().bb_zone_free(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class Engine(object):
    """bb_engine: the batched onQuery handler (lib/server.js:471-507) on one GPU."""

    def __init__(self, dns_domain, datacenter='', recursion=False, snapshot=None, device=0,
                 max_batch=1 << 16, max_batch_bytes=0, ordered=False):
        self._keep = (dns_domain.encode(), datacenter.encode())
        opts = _lib.EngineOpts(self._keep[0], self._keep[1], int(bool(recursion)), device, max_batch,
                               max_batch_bytes, int(bool(ordered)))
        self.ordered = bool(ordered)
        err = ctypes.c_int(0)
        self._h = lib().bb_engine_create(ctypes.byref(opts), ctypes.byref(err))
        if not self._h:
            raise _lib.BinderError(err.value)
        self.dns_domain = dns_domain
        self.max_batch = max_batch
        if snapshot is not None:
            self.load_snapshot(snapshot)

    # -- zone ------------------------------------------------------------------------------
    def load_snapshot(self, snapshot_jsonl, nranks=1, rank=0):
        z = Zone(snapshot_jsonl, self.dns_domain, nranks, rank)
        try:
            self.swap_zone(z)
            return z.stat()
        finally:
            z.close()

    def swap_zone(self, zone):
        check(lib().bb_engine_swap_zone(self._h, zone._h))

    def apply_update(self, zone):
        """After zone.apply(): upload only the changed slots and the arena tail (bb_engine_apply_update)."""
        check(lib().bb_engine_apply_update(self._h, zone._h))

    def set_recursion_filter(self, region_domain, dcs=(), ptr=False):
        """Misses lib/recursion.js:329-344 would refuse without asking anyone are answered REFUSED on the
        device instead of entering the miss list (bb_engine_set_recursion_filter).  None removes it."""
        if region_domain is None:
            check(lib().bb_engine_set_recursion_filter(self._h, None, None, 0, 0))
            return
        arr = (ctypes.c_char_p * max(len(dcs), 1))(*[d.encode('latin-1') for d in dcs])
        check(lib().bb_engine_set_recursion_filter(self._h, region_domain.encode('latin-1'), arr, len(dcs), int(ptr)))

    def is_ready(self):
        return bool(lib().bb_engine_is_ready(self._h))

    def set_kernel_profile(self, profile):
        """Which variant of the resolve kernel batches run on (bb_engine_set_kernel_profile): 'auto' (0), 'small' (1:
        thread per response), 'service' (2: long answers as copy jobs run by the whole tile).  Answers are identical."""
        check(lib().bb_engine_set_kernel_profile(self._h, {'auto': 0, 'small': 1, 'service': 2}.get(profile, profile)))

    def launch_count(self):
        return int(lib().bb_engine_launch_count(self._h))

    # -- host-buffer path (bb_resolve_batch) -------------------------------------------------
    def resolve_batch(self, data, off, seed=0, qidx_base=0, out_cap=None, tcp=False):
        """data: uint8[...] packed packets, off: uint32[n+1] ->
        (out uint8[total], out_off uint32[n+1], out_len uint16[n], status uint8[n], miss uint32[m]);
        response i = out[out_off[i] : out_off[i] + out_len[i]].  tcp: the batch arrived over TCP
        (BB_BATCH_TCP: no UDP size limit)."""
        data = np.ascontiguousarray(data, dtype=np.uint8)
        off = np.ascontiguousarray(off, dtype=np.uint32)
        n = len(off) - 1
        if out_cap is None:
            out_cap = max(4096, min(n * (16384 if tcp else 1232), 0xFFFFFF00))
        out = np.empty(out_cap, dtype=np.uint8)
        out_off = np.zeros(n + 1, dtype=np.uint32)
        out_len = np.zeros(max(n, 1), dtype=np.uint16)
        status = np.zeros(max(n, 1), dtype=np.uint8)
        miss = np.zeros(max(n, 1), dtype=np.uint32)
        n_miss = ctypes.c_uint32(0)
        check(lib().bb_resolve_batch_ex(self._h, data.ctypes.data, off.ctypes.data, n, seed, qidx_base,
                                        out.ctypes.data, out_cap, out_off.ctypes.data, out_len.ctypes.data,
                                        status.ctypes.data, miss.ctypes.data, ctypes.byref(n_miss), 1 if tcp else 0))
        return out[:out_off[n]].copy(), out_off, out_len[:n], status[:n], miss[:n_miss.value].copy()

    # -- recursion relay (bb_relay_batch, lib/recursion.js:287-327) ---------------------------
    def relay_batch(self, q_data, q_off, up_data, up_off, tcp=False, out=None):
        """The replies to forwarded misses: query i (q_data[q_off[i]:q_off[i+1]]) answered from upstream response i
        (up_data[up_off[i]:up_off[i+1]]; empty = the lookup failed) -> (out uint8[total], out_off uint32[n+1],
        out_len uint16[n], status uint8[n]).  tcp: the queries arrived over TCP (no UDP size limit).  out: optional
        (out, out_off, out_len, status) buffers to fill, e.g. pinned ones from bb_host_alloc (then returned as views)."""
        q_data = np.ascontiguousarray(q_data, dtype=np.uint8)
        q_off = np.ascontiguousarray(q_off, dtype=np.uint32)
        up_data = np.ascontiguousarray(up_data, dtype=np.uint8)
        up_off = np.ascontiguousarray(up_off, dtype=np.uint32)
        n = len(q_off) - 1
        if len(up_off) != n + 1:
            raise ValueError('q_off and up_off must have the same length')
        if out is None:
            out_cap = max(4096, min(n * (65535 if tcp else 1200), 0xFFFFFF00))
            out = (np.empty(out_cap, dtype=np.uint8), np.zeros(n + 1, dtype=np.uint32), np.zeros(max(n, 1), dtype=np.uint16),
                   np.zeros(max(n, 1), dtype=np.uint8))
        buf, out_off, out_len, status = out
        check(lib().bb_relay_batch(self._h, q_data.ctypes.data, q_off.ctypes.data, up_data.ctypes.data, up_off.ctypes.data, n,
                                   1 if tcp else 0, buf.ctypes.data, len(buf), out_off.ctypes.data, out_len.ctypes.data,
                                   status.ctypes.data))
        return buf[:out_off[n]].copy(), out_off[:n + 1], out_len[:n], status[:n]

    def relay_device(self, d_q, d_q_off, d_up, d_up_off, n, d_out, out_cap, d_out_off, d_out_len, d_status, d_totals,
                     tcp=False, stream=0):
        """bb_relay_batch_device; pointers are raw device addresses."""
        check(lib().bb_relay_batch_device(self._h, d_q, d_q_off, d_up, d_up_off, n, 1 if tcp else 0, d_out, out_cap, d_out_off,
                                          d_out_len, d_status, d_totals, stream))

    # -- device-buffer path (bb_resolve_batch_device); pointers are raw device addresses ------
    def resolve_device(self, d_pkts, d_off, n, seed, qidx_base, d_out, out_cap, d_out_off, d_out_len, d_status,
                       d_miss, d_totals, stream=0, tcp=False):
        """bb_resolve_batch_device_ex.  tcp: the batch arrived over TCP (BB_BATCH_TCP: no UDP size limit)."""
        check(lib().bb_resolve_batch_device_ex(self._h, d_pkts, d_off, n, seed, qidx_base, d_out, out_cap,
                                               d_out_off, d_out_len, d_status, d_miss, d_totals, stream, 1 if tcp else 0))

    def close(self):
        if getattr(self, '_h', None):
            lib().bb_engine_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:      # interpreter shutdown
            pass
