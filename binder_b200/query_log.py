"""binder's per-query "DNS query" log line (lib/server.js:509-591), written by the server for every response it sends.

The engine renders the parts of the line that the response decides (bb_log_batch, DESIGN.md section 15): the head
`"query":{...},"edns":...` and the body `"rcode":...,"answers":[...],"additional":[...]`.  This module adds the fields
bunyan and the handler add around them, in bunyan's order:

  {"name":"binder","hostname":H,"pid":P,"req_id":<DNS ID>,"client":<address>,"port":"<port>/ipv4"|"/ipv6",<head>,
   "level":30|40,<body>,"latency":<ms>,"timers":{},"msg":"DNS query","time":<ISO 8601>,"v":0}

One line per record, newline-terminated, UTF-8.  level is 40 (warn) when the latency is over 1,000 ms (:511-514).
write() renders a batch's records and writes their lines; write_records() writes the lines of the records a balancer
session kept of its last call (QueryLogRecords: NativeBackend / NativeTcpHub.query_log and their Python models).
"""
import collections
import json
import os
import socket
import threading
import time

import numpy as np

# The records of a balancer session's last call (bb_query_log_records): record i = log[log_off[i]:log_off[i] + log_len[i]],
# its first head_len[i] bytes the head fragment; req_id, client_ip (IPv4 as a u32, 127.0.0.1 = 0x7F000001), client_port
# and, for a TCP hub, session per record (None for a UDP backend); lost = answers whose log call failed.
QueryLogRecords = collections.namedtuple('QueryLogRecords', 'log log_off log_len head_len req_id client_ip client_port session lost')


def ipv4_text(ip):
    ip = int(ip)
    return '%d.%d.%d.%d' % (ip >> 24, (ip >> 16) & 255, (ip >> 8) & 255, ip & 255)


def iso_time(t):
    """Date.prototype.toISOString(): UTC, milliseconds, 'Z'."""
    return time.strftime('%Y-%m-%dT%H:%M:%S', time.gmtime(t)) + '.%03dZ' % (int(t * 1000) % 1000)


class QueryLog(object):
    """A sink for the lines: `stream` is a writable binary stream.  write() may be called from several threads; each
    call writes its lines with one stream.write.  A batch whose log call fails loses its lines and is counted in
    `failed` (the answers have been sent already)."""

    def __init__(self, stream, name='binder', hostname=None, pid=None):
        self.stream = stream
        self._prefix = '{"name":%s,"hostname":%s,"pid":%d,' % (json.dumps(name), json.dumps(hostname or socket.gethostname()),
                                                                os.getpid() if pid is None else pid)
        self._lock = threading.Lock()
        self.lines = 0
        self.failed = 0

    def write(self, resolver, out, out_off, out_len, status, clients, received, sent=None):
        """The lines of one batch of sent responses: (out, out_off, out_len, status) a result set of `resolver` (an
        Engine, or anything with its log_batch), clients[i] = (address, port) of response i, received[i] = when its
        query arrived (time.time()).  sent: when the responses went out (default: now)."""
        status = np.asarray(status)
        if not (status == 0).any():
            return 0
        try:
            log, log_off, log_len, head_len = resolver.log_batch(out, out_off, out_len, status)
        except Exception:                            # BinderError (CUDA): the answers went out, their lines are lost
            self.failed += 1
            return 0
        sent = time.time() if sent is None else sent
        stamp = iso_time(sent)
        log = log.tobytes()
        out = np.asarray(out)
        parts = []
        for i in np.flatnonzero(log_len):
            r = int(out_off[i])
            parts.append(self._line((int(out[r]) << 8) | int(out[r + 1]), clients[i][0], clients[i][1], log, int(log_off[i]),
                                    int(head_len[i]), int(log_len[i]), sent - received[i], stamp))
        return self._emit(parts)

    def write_records(self, records, received, sent=None):
        """The lines of a balancer session's records (a QueryLogRecords), client "a.b.c.d", port "<port>/ipv4".
        received: when each record's query arrived (time.time(); one value for all, or one per record).  sent: when
        the answers went out (default: now).  A record that is empty (its response did not decode) has no line."""
        n = len(records.log_len)
        received = np.broadcast_to(np.asarray(received, dtype=np.float64), (n,))
        sent = time.time() if sent is None else sent
        stamp = iso_time(sent)
        log = np.asarray(records.log, dtype=np.uint8).tobytes()
        parts = [self._line(int(records.req_id[i]), ipv4_text(records.client_ip[i]), int(records.client_port[i]), log,
                            int(records.log_off[i]), int(records.head_len[i]), int(records.log_len[i]), sent - received[i], stamp)
                 for i in np.flatnonzero(records.log_len)]
        return self._emit(parts)

    def _line(self, req_id, addr, port, log, o, hl, ll, wait, stamp):
        """One line: the record log[o:o + ll] (head: its first hl bytes), `wait` seconds after its query arrived."""
        lat = max(0, int(wait * 1000))
        return b''.join((
            ('%s"req_id":%d,"client":%s,"port":"%d/%s",' % (self._prefix, req_id, json.dumps(addr), port,
                                                            'ipv6' if ':' in addr else 'ipv4')).encode(),
            log[o:o + hl], b',"level":%d,' % (40 if lat > 1000 else 30), log[o + hl:o + ll],
            (',"latency":%d,"timers":{},"msg":"DNS query","time":"%s","v":0}\n' % (lat, stamp)).encode()))

    def _emit(self, parts):
        if parts:
            with self._lock:
                self.stream.write(b''.join(parts))
                self.stream.flush()
                self.lines += len(parts)
        return len(parts)
