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
ROUTE_PTR, ROUTE_NONE = 16, 17          # forward routes after the 16 datacenter indices (BB_ROUTE_PTR, BB_ROUTE_NONE)
FORWARD_ROUTES = 18
ERR_CAPACITY = -5                       # BB_ERR_CAPACITY


def ip_u32(addr):
    """Dotted IPv4 -> the host-order integer the forward and match calls take."""
    a, b, c, d = (int(x) for x in addr.split('.'))
    return a << 24 | b << 16 | c << 8 | d


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

    # -- query log (bb_log_batch, lib/server.js:509-591) ---------------------------------------
    def log_batch(self, out, out_off, out_len, status, summary=False, buffers=None):
        """binder's "DNS query" log records of a result set (resolve_batch's or relay_batch's out, out_off, out_len,
        status) -> (log uint8[total], log_off uint32[n+1], log_len uint32[n], head_len uint16[n][, summary uint32[n]]):
        record i = log[log_off[i] : log_off[i] + log_len[i]], its first head_len[i] bytes the head fragment, the rest the
        body (DESIGN.md section 15).  buffers: optional (log, log_off, log_len, head_len, summary) to fill, e.g. pinned
        ones from bb_host_alloc (then returned as views; summary may be None)."""
        out = np.ascontiguousarray(out, dtype=np.uint8)
        out_off = np.ascontiguousarray(out_off, dtype=np.uint32)
        out_len = np.ascontiguousarray(out_len, dtype=np.uint16)
        status = np.ascontiguousarray(status, dtype=np.uint8)
        n = len(status)
        if len(out_off) < n or len(out_len) < n:
            raise ValueError('one offset and one length per status')
        fixed = buffers is not None
        if fixed and summary and buffers[4] is None:
            raise ValueError('summary=True needs a summary buffer in buffers')
        cap = len(buffers[0]) if fixed else max(4096, min(4 * len(out) + 256 * n, 0xFFFFFF00))
        while True:
            if not fixed:
                buffers = (np.empty(cap, dtype=np.uint8), np.zeros(n + 1, dtype=np.uint32), np.zeros(max(n, 1), dtype=np.uint32),
                           np.zeros(max(n, 1), dtype=np.uint16), np.zeros(max(n, 1), dtype=np.uint32) if summary else None)
            log, log_off, log_len, head_len, summ = buffers
            rc = lib().bb_log_batch(self._h, out.ctypes.data, len(out), out_off.ctypes.data, out_len.ctypes.data,
                                    status.ctypes.data, n, log.ctypes.data, len(log), log_off.ctypes.data, log_len.ctypes.data,
                                    head_len.ctypes.data, summ.ctypes.data if summ is not None else None)
            if rc == ERR_CAPACITY and not fixed and cap < 0xFFFFFF00:
                cap = min(cap * 4, 0xFFFFFF00)               # a record can be far longer than its response: try again
                continue
            check(rc)
            break
        res = (log[:log_off[n]].copy(), log_off[:n + 1], log_len[:n], head_len[:n])
        return res + (summ[:n],) if summary else res

    def log_device(self, d_resp, resp_bytes, d_resp_totals, d_out_off, d_out_len, d_status, n, d_log, log_cap, d_log_off,
                   d_log_len, d_head_len, d_summary, d_totals, stream=0):
        """bb_log_batch_device; pointers are raw device addresses (d_resp_totals and d_summary may be 0)."""
        check(lib().bb_log_batch_device(self._h, d_resp, resp_bytes, d_resp_totals or None, d_out_off, d_out_len, d_status, n, d_log,
                                        log_cap, d_log_off, d_log_len, d_head_len, d_summary or None, d_totals, stream))

    # -- recursion forward and match (bb_forward_batch, bb_match_upstreams, lib/recursion.js:253-280,335-354,382-387) --
    def set_recursion_upstreams(self, upstreams):
        """upstreams: [(ipv4 dotted, port, dc index in the filter's list)] (bb_engine_set_recursion_upstreams)."""
        n = len(upstreams)
        ip = np.array([ip_u32(a) for a, _, _ in upstreams] or [0], dtype=np.uint32)
        port = np.array([p for _, p, _ in upstreams] or [0], dtype=np.uint16)
        dc = np.array([d for _, _, d in upstreams] or [0], dtype=np.uint8)
        check(lib().bb_engine_set_recursion_upstreams(self._h, ip.ctypes.data, port.ctypes.data, dc.ctypes.data, n))

    def forward_batch(self, data, off, id_key):
        """Misses data[off[j]:off[j+1]] -> (uq uint8[total], uq_off uint32[n+1], order uint32[n], group_off uint32[19],
        route uint8[n]): upstream query k = uq[uq_off[k]:uq_off[k+1]] is miss order[k]'s; route r's queries are positions
        group_off[r] .. group_off[r+1] (16 = PTR, 17 = nowhere to send)."""
        data = np.ascontiguousarray(data, dtype=np.uint8)
        off = np.ascontiguousarray(off, dtype=np.uint32)
        n = len(off) - 1
        uq = np.empty(max(int(off[n]), 16), dtype=np.uint8)
        uq_off = np.zeros(n + 1, dtype=np.uint32)
        order = np.zeros(max(n, 1), dtype=np.uint32)
        group_off = np.zeros(FORWARD_ROUTES + 1, dtype=np.uint32)
        route = np.zeros(max(n, 1), dtype=np.uint8)
        check(lib().bb_forward_batch(self._h, data.ctypes.data, off.ctypes.data, n, id_key & (2 ** 64 - 1), uq.ctypes.data,
                                     len(uq), uq_off.ctypes.data, order.ctypes.data, group_off.ctypes.data, route.ctypes.data))
        return uq[:uq_off[n]].copy(), uq_off, order[:n], group_off, route[:n]

    def match_upstreams(self, resp, resp_off, src_ip, src_port, q_data, q_off, route, id_key):
        """Received datagrams (packed in arrival order, sources as uint32 IPv4 / uint16 port) against a forward call's
        misses (client queries q_data/q_off and route in miss order) -> (up uint8[total], up_off uint32[n+1]): miss j's
        accepted upstream response, empty when none."""
        resp = np.ascontiguousarray(resp, dtype=np.uint8)
        resp_off = np.ascontiguousarray(resp_off, dtype=np.uint32)
        src_ip = np.ascontiguousarray(src_ip, dtype=np.uint32)
        src_port = np.ascontiguousarray(src_port, dtype=np.uint16)
        q_data = np.ascontiguousarray(q_data, dtype=np.uint8)
        q_off = np.ascontiguousarray(q_off, dtype=np.uint32)
        route = np.ascontiguousarray(route, dtype=np.uint8)
        n_resp, n = len(resp_off) - 1, len(q_off) - 1
        if len(src_ip) != n_resp or len(src_port) != n_resp or len(route) != n:
            raise ValueError('one source per response and one route per miss')
        up = np.empty(max(int(resp_off[n_resp]), 16), dtype=np.uint8)
        up_off = np.zeros(n + 1, dtype=np.uint32)
        check(lib().bb_match_upstreams(self._h, resp.ctypes.data, resp_off.ctypes.data, src_ip.ctypes.data, src_port.ctypes.data,
                                       n_resp, q_data.ctypes.data, q_off.ctypes.data, route.ctypes.data, n,
                                       id_key & (2 ** 64 - 1), up.ctypes.data, len(up), up_off.ctypes.data))
        return up[:up_off[n]].copy(), up_off

    def forward_device(self, d_pkts, d_pkt_off, d_miss_idx, d_resolve_totals, n_cap, id_key, d_uq, uq_cap, d_uq_off, d_order,
                       d_group_off, d_route, d_q, q_cap, d_q_off, d_totals, stream=0):
        """bb_forward_batch_device; pointers are raw device addresses."""
        check(lib().bb_forward_batch_device(self._h, d_pkts, d_pkt_off, d_miss_idx, d_resolve_totals, n_cap, id_key & (2 ** 64 - 1),
                                            d_uq, uq_cap, d_uq_off, d_order, d_group_off, d_route, d_q, q_cap, d_q_off, d_totals,
                                            stream))

    def match_device(self, d_resp, d_resp_off, d_src_ip, d_src_port, n_resp, d_q, d_q_off, d_route, d_forward_totals, n_cap,
                     id_key, d_up, up_cap, d_up_off, d_totals, stream=0):
        """bb_match_upstreams_device; pointers are raw device addresses."""
        check(lib().bb_match_upstreams_device(self._h, d_resp, d_resp_off, d_src_ip, d_src_port, n_resp, d_q, d_q_off, d_route,
                                              d_forward_totals, n_cap, id_key & (2 ** 64 - 1), d_up, up_cap, d_up_off, d_totals,
                                              stream))

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
