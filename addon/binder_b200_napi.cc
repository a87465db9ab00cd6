// N-API shim: binds libbinder_b200.so's C ABI (include/binder_b200.h) into binder's Node.js
// process.  NOT compiled in this repository's image (no node / node_api.h here); it is kept
// thin enough to be read against the header.  Build (on a host with Node >= 10):
//   g++ -std=c++17 -shared -fPIC -I$(node -p "process.execPath+'/../../include/node'") \
//       -I../include binder_b200_napi.cc -L../binder_b200 -lbinder_b200 -o binder_b200.node
//
// JS surface (see INTEGRATION.md):
//   const bb = require('./binder_b200.node');
//   const zone   = bb.zoneBuild(snapshotBuffer, 'dc1.example.com');
//   const engine = bb.engineCreate({dnsDomain, datacenterName, recursion: true, device: 0});
//   bb.engineSwapZone(engine, zone);
//   const r = bb.resolveBatch(engine, pkts /*Buffer*/, pktOff /*Uint32Array n+1*/, seed /*BigInt*/);
//   // r = {out: Buffer, outOff: Uint32Array, outLen: Uint16Array, status: Uint8Array, miss: Uint32Array}
#include <node_api.h>
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <vector>
#include "binder_b200.h"

#define NAPI_OK(call) do { if ((call) != napi_ok) { napi_throw_error(env, nullptr, #call); return nullptr; } } while (0)

static napi_value Throw(napi_env env, int err) {
    napi_throw_error(env, nullptr, err == BB_ERR_CUDA ? bb_last_cuda_error() : bb_strerror(err));
    return nullptr;
}

static napi_value ZoneBuild(napi_env env, napi_callback_info info) {
    size_t argc = 2; napi_value argv[2];
    NAPI_OK(napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr));
    void* data; size_t len; NAPI_OK(napi_get_buffer_info(env, argv[0], &data, &len));
    char dom[256]; size_t dl; NAPI_OK(napi_get_value_string_utf8(env, argv[1], dom, sizeof dom, &dl));
    int err = 0;
    bb_zone* z = bb_zone_build((const char*)data, len, dom, &err);
    if (!z) return Throw(env, err);
    napi_value ext;
    NAPI_OK(napi_create_external(env, z, [](napi_env, void* p, void*) { bb_zone_free((bb_zone*)p); }, nullptr, &ext));
    return ext;
}

static napi_value EngineCreate(napi_env env, napi_callback_info info) {
    size_t argc = 1; napi_value argv[1];
    NAPI_OK(napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr));
    char dom[256] = "", dc[256] = ""; size_t n; napi_value v; bool rec = false; int32_t dev = 0; uint32_t maxb = 1u << 16;
    NAPI_OK(napi_get_named_property(env, argv[0], "dnsDomain", &v)); NAPI_OK(napi_get_value_string_utf8(env, v, dom, sizeof dom, &n));
    if (napi_get_named_property(env, argv[0], "datacenterName", &v) == napi_ok) napi_get_value_string_utf8(env, v, dc, sizeof dc, &n);
    if (napi_get_named_property(env, argv[0], "recursion", &v) == napi_ok) napi_get_value_bool(env, v, &rec);
    if (napi_get_named_property(env, argv[0], "device", &v) == napi_ok) napi_get_value_int32(env, v, &dev);
    if (napi_get_named_property(env, argv[0], "maxBatch", &v) == napi_ok) napi_get_value_uint32(env, v, &maxb);
    bb_engine_opts o; memset(&o, 0, sizeof o);
    o.dns_domain = dom; o.datacenter_name = dc; o.recursion = rec; o.device = dev; o.max_batch = maxb;
    int err = 0;
    bb_engine* e = bb_engine_create(&o, &err);
    if (!e) return Throw(env, err);
    napi_value ext;
    NAPI_OK(napi_create_external(env, e, [](napi_env, void* p, void*) { bb_engine_destroy((bb_engine*)p); }, nullptr, &ext));
    return ext;
}

static napi_value EngineSwapZone(napi_env env, napi_callback_info info) {
    size_t argc = 2; napi_value argv[2];
    NAPI_OK(napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr));
    void *e, *z; NAPI_OK(napi_get_value_external(env, argv[0], &e)); NAPI_OK(napi_get_value_external(env, argv[1], &z));
    int rc = bb_engine_swap_zone((bb_engine*)e, (bb_zone*)z);
    if (rc != BB_OK) return Throw(env, rc);
    return nullptr;
}

// zoneApply(zone, delta: Buffer): watch events as JSON lines (bb_zone_apply)
static napi_value ZoneApply(napi_env env, napi_callback_info info) {
    size_t argc = 2; napi_value argv[2];
    NAPI_OK(napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr));
    void* z; NAPI_OK(napi_get_value_external(env, argv[0], &z));
    void* data; size_t len; NAPI_OK(napi_get_buffer_info(env, argv[1], &data, &len));
    int rc = bb_zone_apply((bb_zone*)z, (const char*)data, len);
    if (rc != BB_OK) return Throw(env, rc);
    return nullptr;
}

// engineApplyUpdate(engine, zone): ship what the deltas changed (bb_engine_apply_update)
static napi_value EngineApplyUpdate(napi_env env, napi_callback_info info) {
    size_t argc = 2; napi_value argv[2];
    NAPI_OK(napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr));
    void *e, *z; NAPI_OK(napi_get_value_external(env, argv[0], &e)); NAPI_OK(napi_get_value_external(env, argv[1], &z));
    int rc = bb_engine_apply_update((bb_engine*)e, (bb_zone*)z);
    if (rc != BB_OK) return Throw(env, rc);
    return nullptr;
}

// engineSetRecursionFilter(engine, regionDomain: string | null, dcNames: string[], ptrForwardable: boolean)
static napi_value EngineSetRecursionFilter(napi_env env, napi_callback_info info) {
    size_t argc = 4; napi_value argv[4];
    NAPI_OK(napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr));
    void* e; NAPI_OK(napi_get_value_external(env, argv[0], &e));
    napi_valuetype t; NAPI_OK(napi_typeof(env, argv[1], &t));
    if (t != napi_string) { int rc0 = bb_engine_set_recursion_filter((bb_engine*)e, nullptr, nullptr, 0, 0); return rc0 == BB_OK ? nullptr : Throw(env, rc0); }
    char dom[256]; size_t dl; NAPI_OK(napi_get_value_string_utf8(env, argv[1], dom, sizeof dom, &dl));
    uint32_t n = 0; NAPI_OK(napi_get_array_length(env, argv[2], &n));
    if (n > 16) return Throw(env, BB_ERR_ARG);
    char names[16][64]; const char* ptrs[16];
    for (uint32_t i = 0; i < n; i++) {
        napi_value v; size_t l; NAPI_OK(napi_get_element(env, argv[2], i, &v));
        NAPI_OK(napi_get_value_string_utf8(env, v, names[i], sizeof names[i], &l)); ptrs[i] = names[i];
    }
    bool ptr = false; napi_get_value_bool(env, argv[3], &ptr);
    int rc = bb_engine_set_recursion_filter((bb_engine*)e, dom, ptrs, n, ptr ? 1 : 0);
    if (rc != BB_OK) return Throw(env, rc);
    return nullptr;
}

// resolveBatch(engine, pkts: Buffer, pktOff: Uint32Array(n+1), seed: BigInt[, tcp: boolean]) -> result object
static napi_value ResolveBatch(napi_env env, napi_callback_info info) {
    size_t argc = 5; napi_value argv[5];
    NAPI_OK(napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr));
    bool tcp = false;                              // optional 5th argument: the batch arrived over TCP
    if (argc > 4) napi_get_value_bool(env, argv[4], &tcp);
    void* e; NAPI_OK(napi_get_value_external(env, argv[0], &e));
    void* pk; size_t pklen; NAPI_OK(napi_get_buffer_info(env, argv[1], &pk, &pklen));
    napi_typedarray_type tt; size_t offn; void* offp; napi_value ab; size_t bo;
    NAPI_OK(napi_get_typedarray_info(env, argv[2], &tt, &offn, &offp, &ab, &bo));
    uint64_t seed = 0; bool lossless; napi_get_value_bigint_uint64(env, argv[3], &seed, &lossless);
    // pktOff: at least one entry, ascending, ending inside the pkts Buffer (the engine trusts only what it can check cheaply)
    if (tt != napi_uint32_array || offn < 1 || offn > (1u << 22) + 1) return Throw(env, BB_ERR_ARG);
    {
        const uint32_t* po = (const uint32_t*)offp;
        for (size_t i = 1; i < offn; i++) if (po[i] < po[i - 1]) return Throw(env, BB_ERR_ARG);
        if (po[offn - 1] > pklen) return Throw(env, BB_ERR_ARG);
    }
    const uint32_t n = (uint32_t)offn - 1;
    const uint32_t cap = n * (tcp ? 16384u : 1232u);
    void *out, *oo, *ol, *st, *ms; napi_value o_out, a_oo, a_ol, a_st, a_ms, t_oo, t_ol, t_st, t_ms;
    NAPI_OK(napi_create_buffer(env, cap, &out, &o_out));
    NAPI_OK(napi_create_arraybuffer(env, (n + 1) * 4, &oo, &a_oo)); NAPI_OK(napi_create_typedarray(env, napi_uint32_array, n + 1, a_oo, 0, &t_oo));
    NAPI_OK(napi_create_arraybuffer(env, n * 2, &ol, &a_ol));       NAPI_OK(napi_create_typedarray(env, napi_uint16_array, n, a_ol, 0, &t_ol));
    NAPI_OK(napi_create_arraybuffer(env, n, &st, &a_st));           NAPI_OK(napi_create_typedarray(env, napi_uint8_array, n, a_st, 0, &t_st));
    NAPI_OK(napi_create_arraybuffer(env, n * 4, &ms, &a_ms));
    uint32_t nmiss = 0;
    int rc = bb_resolve_batch_ex((bb_engine*)e, (const uint8_t*)pk, (const uint32_t*)offp, n, seed, 0, (uint8_t*)out, cap,
                                 (uint32_t*)oo, (uint16_t*)ol, (uint8_t*)st, (uint32_t*)ms, &nmiss, tcp ? BB_BATCH_TCP : 0u);
    if (rc != BB_OK) return Throw(env, rc);
    NAPI_OK(napi_create_typedarray(env, napi_uint32_array, nmiss, a_ms, 0, &t_ms));
    napi_value res; NAPI_OK(napi_create_object(env, &res));
    napi_set_named_property(env, res, "out", o_out);   napi_set_named_property(env, res, "outOff", t_oo);
    napi_set_named_property(env, res, "outLen", t_ol); napi_set_named_property(env, res, "status", t_st);
    napi_set_named_property(env, res, "miss", t_ms);
    return res;
}

// relayBatch(engine, pkts: Buffer, pktOff: Uint32Array(n+1), upstream: Buffer, upOff: Uint32Array(n+1)[, tcp: boolean])
//   -> {out, outOff, outLen, status}: the replies Recursion.prototype.resolve's respond() builds from the upstream's
//   answers (lib/recursion.js:287-327, bb_relay_batch); an empty upstream (upOff[i] == upOff[i+1]) = the lookup failed
static bool check_off(napi_env env, napi_value v, size_t bytes, const uint32_t** off, size_t* n) {
    napi_typedarray_type tt; void* p; napi_value ab; size_t bo;
    if (napi_get_typedarray_info(env, v, &tt, n, &p, &ab, &bo) != napi_ok || tt != napi_uint32_array || *n < 1 || *n > (1u << 22) + 1) return false;
    *off = (const uint32_t*)p;
    for (size_t i = 1; i < *n; i++) if ((*off)[i] < (*off)[i - 1]) return false;
    return (*off)[*n - 1] <= bytes;
}
static napi_value RelayBatch(napi_env env, napi_callback_info info) {
    size_t argc = 6; napi_value argv[6];
    NAPI_OK(napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr));
    bool tcp = false;
    if (argc > 5) napi_get_value_bool(env, argv[5], &tcp);
    void* e; NAPI_OK(napi_get_value_external(env, argv[0], &e));
    void* pk; size_t pklen; NAPI_OK(napi_get_buffer_info(env, argv[1], &pk, &pklen));
    void* up; size_t uplen; NAPI_OK(napi_get_buffer_info(env, argv[3], &up, &uplen));
    const uint32_t *qo, *uo; size_t qn, un;
    if (!check_off(env, argv[2], pklen, &qo, &qn) || !check_off(env, argv[4], uplen, &uo, &un) || qn != un) return Throw(env, BB_ERR_ARG);
    const uint32_t n = (uint32_t)qn - 1;
    const uint64_t cap64 = (uint64_t)n * (tcp ? 65535u : 1200u);
    const uint32_t cap = cap64 > 0xFFFFFF00u ? 0xFFFFFF00u : (uint32_t)cap64;
    void *out, *oo, *ol, *st; napi_value o_out, a_oo, a_ol, a_st, t_oo, t_ol, t_st;
    NAPI_OK(napi_create_buffer(env, cap, &out, &o_out));
    NAPI_OK(napi_create_arraybuffer(env, (n + 1) * 4, &oo, &a_oo)); NAPI_OK(napi_create_typedarray(env, napi_uint32_array, n + 1, a_oo, 0, &t_oo));
    NAPI_OK(napi_create_arraybuffer(env, n * 2, &ol, &a_ol));       NAPI_OK(napi_create_typedarray(env, napi_uint16_array, n, a_ol, 0, &t_ol));
    NAPI_OK(napi_create_arraybuffer(env, n, &st, &a_st));           NAPI_OK(napi_create_typedarray(env, napi_uint8_array, n, a_st, 0, &t_st));
    int rc = bb_relay_batch((bb_engine*)e, (const uint8_t*)pk, qo, (const uint8_t*)up, uo, n, tcp ? BB_BATCH_TCP : 0u, (uint8_t*)out, cap,
                            (uint32_t*)oo, (uint16_t*)ol, (uint8_t*)st);
    if (rc != BB_OK) return Throw(env, rc);
    napi_value res; NAPI_OK(napi_create_object(env, &res));
    napi_set_named_property(env, res, "out", o_out);   napi_set_named_property(env, res, "outOff", t_oo);
    napi_set_named_property(env, res, "outLen", t_ol); napi_set_named_property(env, res, "status", t_st);
    return res;
}

// logBatch(engine, out: Buffer, outOff: Uint32Array, outLen: Uint16Array(n), status: Uint8Array(n))
//   -> {log: Buffer, logOff: Uint32Array(n+1), logLen: Uint32Array(n), headLen: Uint16Array(n), summary: Uint32Array(n)}:
//   binder's "DNS query" record of each response of a resolveBatch / relayBatch result (bb_log_batch, lib/server.js:509-591).
//   Record i = log[logOff[i] .. +logLen[i]); its first headLen[i] bytes are the head, the rest the body (DESIGN.md section 15).
static napi_value LogBatch(napi_env env, napi_callback_info info) {
    size_t argc = 5; napi_value argv[5];
    NAPI_OK(napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr));
    if (argc < 5) return Throw(env, BB_ERR_ARG);
    void* e; NAPI_OK(napi_get_value_external(env, argv[0], &e));
    void* out; size_t outlen; NAPI_OK(napi_get_buffer_info(env, argv[1], &out, &outlen));
    napi_typedarray_type t1, t2, t3; size_t n1, n2, n3; void *p1, *p2, *p3; napi_value ab; size_t bo;
    NAPI_OK(napi_get_typedarray_info(env, argv[2], &t1, &n1, &p1, &ab, &bo));
    NAPI_OK(napi_get_typedarray_info(env, argv[3], &t2, &n2, &p2, &ab, &bo));
    NAPI_OK(napi_get_typedarray_info(env, argv[4], &t3, &n3, &p3, &ab, &bo));
    // the offsets and lengths need not be checked here: the kernel bounds-checks every response against outlen
    if (t1 != napi_uint32_array || t2 != napi_uint16_array || t3 != napi_uint8_array || n1 < n3 || n2 < n3 || n3 > (1u << 22) ||
        outlen > 0xFFFFFFFFu)
        return Throw(env, BB_ERR_ARG);
    const uint32_t n = (uint32_t)n3;
    void *lo, *ll, *hl, *sm; napi_value a_lo, a_ll, a_hl, a_sm, t_lo, t_ll, t_hl, t_sm;
    NAPI_OK(napi_create_arraybuffer(env, ((size_t)n + 1) * 4, &lo, &a_lo)); NAPI_OK(napi_create_typedarray(env, napi_uint32_array, n + 1, a_lo, 0, &t_lo));
    NAPI_OK(napi_create_arraybuffer(env, (size_t)n * 4, &ll, &a_ll));       NAPI_OK(napi_create_typedarray(env, napi_uint32_array, n, a_ll, 0, &t_ll));
    NAPI_OK(napi_create_arraybuffer(env, (size_t)n * 2, &hl, &a_hl));       NAPI_OK(napi_create_typedarray(env, napi_uint16_array, n, a_hl, 0, &t_hl));
    NAPI_OK(napi_create_arraybuffer(env, (size_t)n * 4, &sm, &a_sm));       NAPI_OK(napi_create_typedarray(env, napi_uint32_array, n, a_sm, 0, &t_sm));
    // a record can be far longer than its response: start at 4 bytes per response byte + 256 per record, grow on overflow
    uint64_t cap = std::max<uint64_t>(4096, std::min<uint64_t>(4ull * outlen + 256ull * n, 0xFFFFFF00u));
    for (;;) {
        void* lg; napi_value b_lg;
        NAPI_OK(napi_create_buffer(env, (size_t)cap, &lg, &b_lg));
        int rc = bb_log_batch((bb_engine*)e, (const uint8_t*)out, (uint32_t)outlen, (const uint32_t*)p1, (const uint16_t*)p2,
                              (const uint8_t*)p3, n, (uint8_t*)lg, (uint32_t)cap, (uint32_t*)lo, (uint32_t*)ll, (uint16_t*)hl, (uint32_t*)sm);
        if (rc == BB_ERR_CAPACITY && cap < 0xFFFFFF00u) { cap = std::min<uint64_t>(cap * 4, 0xFFFFFF00u); continue; }
        if (rc != BB_OK) return Throw(env, rc);
        napi_value res; NAPI_OK(napi_create_object(env, &res));
        napi_set_named_property(env, res, "log", b_lg);      napi_set_named_property(env, res, "logOff", t_lo);
        napi_set_named_property(env, res, "logLen", t_ll);   napi_set_named_property(env, res, "headLen", t_hl);
        napi_set_named_property(env, res, "summary", t_sm);
        return res;
    }
}

// engineSetRecursionUpstreams(engine, ip: Uint32Array, port: Uint16Array, dc: Uint8Array)   (bb_engine_set_recursion_upstreams;
//   ip and port in host byte order, dc = index in the filter's datacenter list)
static napi_value EngineSetRecursionUpstreams(napi_env env, napi_callback_info info) {
    size_t argc = 4; napi_value argv[4];
    NAPI_OK(napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr));
    void* e; NAPI_OK(napi_get_value_external(env, argv[0], &e));
    napi_typedarray_type t1, t2, t3; size_t n1, n2, n3; void *p1, *p2, *p3; napi_value ab; size_t bo;
    NAPI_OK(napi_get_typedarray_info(env, argv[1], &t1, &n1, &p1, &ab, &bo));
    NAPI_OK(napi_get_typedarray_info(env, argv[2], &t2, &n2, &p2, &ab, &bo));
    NAPI_OK(napi_get_typedarray_info(env, argv[3], &t3, &n3, &p3, &ab, &bo));
    if (t1 != napi_uint32_array || t2 != napi_uint16_array || t3 != napi_uint8_array || n1 != n2 || n1 != n3) return Throw(env, BB_ERR_ARG);
    int rc = bb_engine_set_recursion_upstreams((bb_engine*)e, (const uint32_t*)p1, (const uint16_t*)p2, (const uint8_t*)p3, (uint32_t)n1);
    if (rc != BB_OK) return Throw(env, rc);
    return nullptr;
}

// forwardBatch(engine, pkts: Buffer, pktOff: Uint32Array(n+1), idKey: BigInt)
//   -> {uq: Buffer, uqOff: Uint32Array(n+1), order: Uint32Array(n), groupOff: Uint32Array(19), route: Uint8Array(n)}:
//   the upstream queries of the misses, grouped by datacenter (bb_forward_batch); draw a fresh idKey for every call
static napi_value ForwardBatch(napi_env env, napi_callback_info info) {
    size_t argc = 4; napi_value argv[4];
    NAPI_OK(napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr));
    void* e; NAPI_OK(napi_get_value_external(env, argv[0], &e));
    void* pk; size_t pklen; NAPI_OK(napi_get_buffer_info(env, argv[1], &pk, &pklen));
    const uint32_t* po; size_t pn;
    if (!check_off(env, argv[2], pklen, &po, &pn) || pn - 1 > BB_FORWARD_MAX) return Throw(env, BB_ERR_ARG);
    uint64_t key = 0; bool lossless; NAPI_OK(napi_get_value_bigint_uint64(env, argv[3], &key, &lossless));
    const uint32_t n = (uint32_t)pn - 1, cap = po[n];
    void *uq, *uo, *od, *go, *rt; napi_value b_uq, a_uo, a_od, a_go, a_rt, t_uo, t_od, t_go, t_rt;
    NAPI_OK(napi_create_buffer(env, cap ? cap : 1, &uq, &b_uq));
    NAPI_OK(napi_create_arraybuffer(env, (n + 1) * 4, &uo, &a_uo)); NAPI_OK(napi_create_typedarray(env, napi_uint32_array, n + 1, a_uo, 0, &t_uo));
    NAPI_OK(napi_create_arraybuffer(env, n * 4, &od, &a_od));       NAPI_OK(napi_create_typedarray(env, napi_uint32_array, n, a_od, 0, &t_od));
    NAPI_OK(napi_create_arraybuffer(env, (BB_ROUTE_NONE + 2) * 4, &go, &a_go));
    NAPI_OK(napi_create_typedarray(env, napi_uint32_array, BB_ROUTE_NONE + 2, a_go, 0, &t_go));
    NAPI_OK(napi_create_arraybuffer(env, n, &rt, &a_rt));           NAPI_OK(napi_create_typedarray(env, napi_uint8_array, n, a_rt, 0, &t_rt));
    int rc = bb_forward_batch((bb_engine*)e, (const uint8_t*)pk, po, n, key, (uint8_t*)uq, cap, (uint32_t*)uo, (uint32_t*)od, (uint32_t*)go,
                              (uint8_t*)rt);
    if (rc != BB_OK) return Throw(env, rc);
    napi_value res; NAPI_OK(napi_create_object(env, &res));
    napi_set_named_property(env, res, "uq", b_uq);         napi_set_named_property(env, res, "uqOff", t_uo);
    napi_set_named_property(env, res, "order", t_od);      napi_set_named_property(env, res, "groupOff", t_go);
    napi_set_named_property(env, res, "route", t_rt);
    return res;
}

// matchUpstreams(engine, resp: Buffer, respOff: Uint32Array(m+1), srcIp: Uint32Array(m), srcPort: Uint16Array(m),
//                pkts: Buffer, pktOff: Uint32Array(n+1), route: Uint8Array(n), idKey: BigInt)
//   -> {up: Buffer, upOff: Uint32Array(n+1)}: each miss's accepted upstream response, relayBatch's upstream input
//   (bb_match_upstreams); pkts / route are the forwardBatch call's misses and routes, in miss order
static napi_value MatchUpstreams(napi_env env, napi_callback_info info) {
    size_t argc = 9; napi_value argv[9];
    NAPI_OK(napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr));
    void* e; NAPI_OK(napi_get_value_external(env, argv[0], &e));
    void* rs; size_t rslen; NAPI_OK(napi_get_buffer_info(env, argv[1], &rs, &rslen));
    void* pk; size_t pklen; NAPI_OK(napi_get_buffer_info(env, argv[5], &pk, &pklen));
    const uint32_t *ro, *po; size_t rn, pn;
    if (!check_off(env, argv[2], rslen, &ro, &rn) || !check_off(env, argv[6], pklen, &po, &pn)) return Throw(env, BB_ERR_ARG);
    napi_typedarray_type ti, tp, tr; size_t ni, np_, nr; void *pi, *pp, *pr; napi_value ab; size_t bo;
    NAPI_OK(napi_get_typedarray_info(env, argv[3], &ti, &ni, &pi, &ab, &bo));
    NAPI_OK(napi_get_typedarray_info(env, argv[4], &tp, &np_, &pp, &ab, &bo));
    NAPI_OK(napi_get_typedarray_info(env, argv[7], &tr, &nr, &pr, &ab, &bo));
    if (ti != napi_uint32_array || tp != napi_uint16_array || tr != napi_uint8_array || ni != rn - 1 || np_ != rn - 1 || nr != pn - 1)
        return Throw(env, BB_ERR_ARG);
    uint64_t key = 0; bool lossless; NAPI_OK(napi_get_value_bigint_uint64(env, argv[8], &key, &lossless));
    const uint32_t m = (uint32_t)rn - 1, n = (uint32_t)pn - 1, cap = ro[m];
    void *up, *uo; napi_value b_up, a_uo, t_uo;
    NAPI_OK(napi_create_buffer(env, cap ? cap : 1, &up, &b_up));
    NAPI_OK(napi_create_arraybuffer(env, (n + 1) * 4, &uo, &a_uo)); NAPI_OK(napi_create_typedarray(env, napi_uint32_array, n + 1, a_uo, 0, &t_uo));
    int rc = bb_match_upstreams((bb_engine*)e, (const uint8_t*)rs, ro, (const uint32_t*)pi, (const uint16_t*)pp, m, (const uint8_t*)pk, po,
                                (const uint8_t*)pr, n, key, (uint8_t*)up, cap, (uint32_t*)uo);
    if (rc != BB_OK) return Throw(env, rc);
    napi_value res; NAPI_OK(napi_create_object(env, &res));
    napi_set_named_property(env, res, "up", b_up); napi_set_named_property(env, res, "upOff", t_uo);
    return res;
}

// ---- TCP proxy sessions from mname-balancer (bb_tcp_hub): route a new AF_UNIX connection whose first frame is
// INBOUND_TCP here.  Session ids travel as Uint32Array(1), counters as BigUint64Array.
//   tcpHubCreate(engine, maxBatch) -> hub          tcpHubOpen(hub) -> Uint32Array [session]
//   tcpHubFeed(hub, session, Buffer)  (throws on a protocol error: the session reads nothing more; drain it, then close)
//   tcpHubEof(hub, session)          tcpHubFlush(hub, seed: BigInt) -> misses {pkts: Buffer, pktOff: Uint32Array, session: Uint32Array}
//   tcpHubOutput(hub, session) -> {out: Buffer, closable: Uint8Array(1)}     tcpHubConsume(hub, session, nBytes)
//   tcpHubClose(hub, session)        tcpHubRelay(hub, pkts, pktOff, upstream, upOff, sessions: Uint32Array)
//   tcpHubStats(hub) -> BigUint64Array(13)   (bb_tcp_hub_stat 0..12)
//   tcpHubSetQueryLog(hub, on: bool)   tcpHubQueryLog(hub, which: 0 last flush | 1 last relay) -> the "DNS query" log records
//       of the answers appended: {log: Buffer, logOff, logLen: Uint32Array, headLen, reqId: Uint16Array, clientIp,
//       clientPort, session: Uint32Array, lost: Uint32Array(1)}   (bb_query_log_tcp_hub; record i = log[logOff[i] ..
//       logOff[i] + logLen[i]), its first headLen[i] bytes the head fragment)
static napi_value U32Array(napi_env env, const uint32_t* src, size_t n) {
    void* p; napi_value ab, t;
    if (napi_create_arraybuffer(env, n * 4, &p, &ab) != napi_ok || napi_create_typedarray(env, napi_uint32_array, n, ab, 0, &t) != napi_ok) return nullptr;
    if (n) memcpy(p, src, n * 4);
    return t;
}
static napi_value CopyBuffer(napi_env env, const uint8_t* src, size_t n) {
    void* p; napi_value b;
    if (napi_create_buffer(env, n, &p, &b) != napi_ok) return nullptr;
    if (n) memcpy(p, src, n);
    return b;
}
static napi_value U16Array(napi_env env, const uint16_t* src, size_t n) {
    void* p; napi_value ab, t;
    if (napi_create_arraybuffer(env, n * 2, &p, &ab) != napi_ok || napi_create_typedarray(env, napi_uint16_array, n, ab, 0, &t) != napi_ok) return nullptr;
    if (n) memcpy(p, src, n * 2);
    return t;
}
// bb_query_log_records -> the object of backendQueryLog / tcpHubQueryLog (copies: the session's arrays change with its next call)
static napi_value QueryLogObject(napi_env env, const bb_query_log_records& r) {
    size_t end = 0;
    for (uint32_t i = 0; i < r.n; i++) end = std::max(end, (size_t)r.log_off[i] + r.log_len[i]);
    napi_value res;
    if (napi_create_object(env, &res) != napi_ok) return nullptr;
    napi_set_named_property(env, res, "log", CopyBuffer(env, r.log, end));
    napi_set_named_property(env, res, "logOff", U32Array(env, r.log_off, r.n));
    napi_set_named_property(env, res, "logLen", U32Array(env, r.log_len, r.n));
    napi_set_named_property(env, res, "headLen", U16Array(env, r.head_len, r.n));
    napi_set_named_property(env, res, "reqId", U16Array(env, r.req_id, r.n));
    napi_set_named_property(env, res, "clientIp", U32Array(env, r.client_ip, r.n));
    napi_set_named_property(env, res, "clientPort", U32Array(env, r.client_port, r.n));
    if (r.session) napi_set_named_property(env, res, "session", U32Array(env, r.session, r.n));
    napi_set_named_property(env, res, "lost", U32Array(env, &r.lost, 1));
    return res;
}
static napi_value TcpHubCreate(napi_env env, napi_callback_info info) {
    size_t argc = 2; napi_value argv[2];
    NAPI_OK(napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr));
    void* e; NAPI_OK(napi_get_value_external(env, argv[0], &e));
    uint32_t maxb = 4096; if (argc > 1) napi_get_value_uint32(env, argv[1], &maxb);
    int err = 0;
    bb_tcp_hub* h = bb_tcp_hub_create((bb_engine*)e, maxb, &err);
    if (!h) return Throw(env, err);
    napi_value ext;
    NAPI_OK(napi_create_external(env, h, [](napi_env, void* p, void*) { bb_tcp_hub_destroy((bb_tcp_hub*)p); }, nullptr, &ext));
    return ext;
}
static napi_value TcpHubOpen(napi_env env, napi_callback_info info) {
    size_t argc = 1; napi_value argv[1];
    NAPI_OK(napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr));
    void* h; NAPI_OK(napi_get_value_external(env, argv[0], &h));
    uint32_t sid = 0; int rc = bb_tcp_hub_open((bb_tcp_hub*)h, &sid);
    if (rc != BB_OK) return Throw(env, rc);
    return U32Array(env, &sid, 1);
}
// hub and session of a tcpHub* call (argv[0], argv[1])
static bool HubSession(napi_env env, napi_value* argv, void** h, uint32_t* sid) {
    return napi_get_value_external(env, argv[0], h) == napi_ok && napi_get_value_uint32(env, argv[1], sid) == napi_ok;
}
static napi_value TcpHubFeed(napi_env env, napi_callback_info info) {
    size_t argc = 3; napi_value argv[3];
    NAPI_OK(napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr));
    void* h; uint32_t sid; if (!HubSession(env, argv, &h, &sid)) return Throw(env, BB_ERR_ARG);
    void* data; size_t len; NAPI_OK(napi_get_buffer_info(env, argv[2], &data, &len));
    int rc = bb_tcp_hub_feed((bb_tcp_hub*)h, sid, (const uint8_t*)data, len);
    if (rc != BB_OK) return Throw(env, rc);
    return nullptr;
}
static napi_value TcpHubEof(napi_env env, napi_callback_info info) {
    size_t argc = 2; napi_value argv[2];
    NAPI_OK(napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr));
    void* h; uint32_t sid; if (!HubSession(env, argv, &h, &sid)) return Throw(env, BB_ERR_ARG);
    int rc = bb_tcp_hub_eof((bb_tcp_hub*)h, sid);
    if (rc != BB_OK) return Throw(env, rc);
    return nullptr;
}
static napi_value TcpHubFlush(napi_env env, napi_callback_info info) {
    size_t argc = 2; napi_value argv[2];
    NAPI_OK(napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr));
    void* h; NAPI_OK(napi_get_value_external(env, argv[0], &h));
    uint64_t seed = 0; bool lossless; napi_get_value_bigint_uint64(env, argv[1], &seed, &lossless);
    bb_tcp_hub_misses m; memset(&m, 0, sizeof m);
    int rc = bb_tcp_hub_flush((bb_tcp_hub*)h, seed, &m);
    if (rc == BB_ERR_ARG) return Throw(env, rc);              // a failed batch is counted (tcpHubStats), not thrown
    napi_value res; NAPI_OK(napi_create_object(env, &res));
    const uint32_t zero = 0;
    napi_set_named_property(env, res, "pkts", CopyBuffer(env, m.pkts, m.n ? m.pkt_off[m.n] : 0));
    napi_set_named_property(env, res, "pktOff", U32Array(env, m.n ? m.pkt_off : &zero, (size_t)m.n + 1));
    napi_set_named_property(env, res, "session", U32Array(env, m.session, m.n));
    return res;
}
static napi_value TcpHubOutput(napi_env env, napi_callback_info info) {
    size_t argc = 2; napi_value argv[2];
    NAPI_OK(napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr));
    void* h; uint32_t sid; if (!HubSession(env, argv, &h, &sid)) return Throw(env, BB_ERR_ARG);
    const uint8_t* out; size_t len; int closable = 0;
    int rc = bb_tcp_hub_output((bb_tcp_hub*)h, sid, &out, &len, &closable);
    if (rc != BB_OK) return Throw(env, rc);
    void* cp; napi_value ab, cl, res;
    NAPI_OK(napi_create_arraybuffer(env, 1, &cp, &ab)); NAPI_OK(napi_create_typedarray(env, napi_uint8_array, 1, ab, 0, &cl));
    *(uint8_t*)cp = (uint8_t)closable;
    NAPI_OK(napi_create_object(env, &res));
    napi_set_named_property(env, res, "out", CopyBuffer(env, out, len));
    napi_set_named_property(env, res, "closable", cl);
    return res;
}
static napi_value TcpHubConsume(napi_env env, napi_callback_info info) {
    size_t argc = 3; napi_value argv[3];
    NAPI_OK(napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr));
    void* h; uint32_t sid, n; if (!HubSession(env, argv, &h, &sid)) return Throw(env, BB_ERR_ARG);
    NAPI_OK(napi_get_value_uint32(env, argv[2], &n));
    int rc = bb_tcp_hub_consume((bb_tcp_hub*)h, sid, n);
    if (rc != BB_OK) return Throw(env, rc);
    return nullptr;
}
static napi_value TcpHubClose(napi_env env, napi_callback_info info) {
    size_t argc = 2; napi_value argv[2];
    NAPI_OK(napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr));
    void* h; uint32_t sid; if (!HubSession(env, argv, &h, &sid)) return Throw(env, BB_ERR_ARG);
    int rc = bb_tcp_hub_close((bb_tcp_hub*)h, sid);
    if (rc != BB_OK) return Throw(env, rc);
    return nullptr;
}
static napi_value TcpHubRelay(napi_env env, napi_callback_info info) {
    size_t argc = 6; napi_value argv[6];
    NAPI_OK(napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr));
    void* h; NAPI_OK(napi_get_value_external(env, argv[0], &h));
    void* pk; size_t pklen; NAPI_OK(napi_get_buffer_info(env, argv[1], &pk, &pklen));
    void* up; size_t uplen; NAPI_OK(napi_get_buffer_info(env, argv[3], &up, &uplen));
    const uint32_t *qo, *uo; size_t qn, un;
    if (!check_off(env, argv[2], pklen, &qo, &qn) || !check_off(env, argv[4], uplen, &uo, &un) || qn != un) return Throw(env, BB_ERR_ARG);
    napi_typedarray_type tt; size_t sn; void* sp; napi_value ab; size_t bo;
    if (napi_get_typedarray_info(env, argv[5], &tt, &sn, &sp, &ab, &bo) != napi_ok || tt != napi_uint32_array || sn != qn - 1)
        return Throw(env, BB_ERR_ARG);
    int rc = bb_tcp_hub_relay((bb_tcp_hub*)h, (const uint8_t*)pk, qo, (const uint8_t*)up, uo, (const uint32_t*)sp, (uint32_t)sn);
    if (rc == BB_ERR_ARG) return Throw(env, rc);              // a failed batch is counted, not thrown
    return nullptr;
}
static napi_value TcpHubStats(napi_env env, napi_callback_info info) {
    size_t argc = 1; napi_value argv[1];
    NAPI_OK(napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr));
    void* h; NAPI_OK(napi_get_value_external(env, argv[0], &h));
    void* p; napi_value ab, t;
    NAPI_OK(napi_create_arraybuffer(env, 13 * 8, &p, &ab)); NAPI_OK(napi_create_typedarray(env, napi_biguint64_array, 13, ab, 0, &t));
    for (int i = 0; i < 13; i++) ((uint64_t*)p)[i] = bb_tcp_hub_stat((const bb_tcp_hub*)h, i);
    return t;
}
static napi_value TcpHubSetQueryLog(napi_env env, napi_callback_info info) {
    size_t argc = 2; napi_value argv[2];
    NAPI_OK(napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr));
    void* h; NAPI_OK(napi_get_value_external(env, argv[0], &h));
    bool on = false; NAPI_OK(napi_get_value_bool(env, argv[1], &on));
    const int rc = bb_query_log_tcp_hub_enable((bb_tcp_hub*)h, on ? 1 : 0);
    return rc == BB_OK ? nullptr : Throw(env, rc);
}
static napi_value TcpHubQueryLog(napi_env env, napi_callback_info info) {
    size_t argc = 2; napi_value argv[2];
    NAPI_OK(napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr));
    void* h; NAPI_OK(napi_get_value_external(env, argv[0], &h));
    uint32_t which = 0; NAPI_OK(napi_get_value_uint32(env, argv[1], &which));
    bb_query_log_records r;
    const int rc = bb_query_log_tcp_hub((const bb_tcp_hub*)h, (int)std::min(which, 2u), &r);
    return rc == BB_OK ? QueryLogObject(env, r) : Throw(env, rc);
}

// A native balancer UDP session (bb_backend_*, include/binder_b200.h):
//   backendCreate(engine, maxBatch = 16384) -> session
//   backendFeed(session, bytes: Buffer, seed: BigInt) -> {out: Buffer (frames to write), pkts: Buffer, pktOff: Uint32Array,
//       srcIp: Uint32Array, srcPort: Uint32Array}   (the misses, for the host's recursion; a failed batch is counted, not thrown)
//   backendRelay(session, pkts, pktOff, upstream, upOff, dstIp: Uint32Array, dstPort: Uint32Array) -> Buffer (OUTBOUND_UDP
//       frames of the misses' replies; a failed batch is counted, not thrown)
//   backendStats(session) -> BigUint64Array(10)   (bb_backend_stat 0..9)
//   backendSetQueryLog(session, on: bool)   backendQueryLog(session, which: 0 last feed | 1 last relay) -> the "DNS query"
//       log records of the frames sent, one per OUTBOUND_UDP frame in order: {log: Buffer, logOff, logLen: Uint32Array,
//       headLen, reqId: Uint16Array, clientIp, clientPort: Uint32Array, lost: Uint32Array(1)}   (bb_query_log_backend)
//   backendDestroy(session)   (also done when the session is garbage-collected)
struct BackendRef { bb_backend* b; };
static bb_backend* BackendOf(napi_env env, napi_value v) {
    void* p = nullptr;
    if (napi_get_value_external(env, v, &p) != napi_ok || !p) return nullptr;
    return ((BackendRef*)p)->b;
}
static napi_value BackendCreate(napi_env env, napi_callback_info info) {
    size_t argc = 2; napi_value argv[2];
    NAPI_OK(napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr));
    void* e; NAPI_OK(napi_get_value_external(env, argv[0], &e));
    uint32_t maxb = 1u << 14; if (argc > 1) napi_get_value_uint32(env, argv[1], &maxb);
    int err = 0;
    bb_backend* b = bb_backend_create((bb_engine*)e, maxb, &err);
    if (!b) return Throw(env, err);
    napi_value ext;
    NAPI_OK(napi_create_external(env, new BackendRef{b}, [](napi_env, void* p, void*) {
        bb_backend_destroy(((BackendRef*)p)->b); delete (BackendRef*)p; }, nullptr, &ext));
    return ext;
}
static napi_value BackendFeed(napi_env env, napi_callback_info info) {
    size_t argc = 3; napi_value argv[3];
    NAPI_OK(napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr));
    bb_backend* b = BackendOf(env, argv[0]); if (!b) return Throw(env, BB_ERR_ARG);
    void* data; size_t len; NAPI_OK(napi_get_buffer_info(env, argv[1], &data, &len));
    uint64_t seed = 0; bool lossless; napi_get_value_bigint_uint64(env, argv[2], &seed, &lossless);
    const uint8_t* out = nullptr; size_t out_len = 0; bb_backend_misses m; memset(&m, 0, sizeof m);
    int rc = bb_backend_feed(b, (const uint8_t*)data, len, seed, &out, &out_len, &m);
    if (rc == BB_ERR_ARG) return Throw(env, rc);
    napi_value res; NAPI_OK(napi_create_object(env, &res));
    const uint32_t zero = 0;
    napi_set_named_property(env, res, "out", CopyBuffer(env, out, out_len));
    napi_set_named_property(env, res, "pkts", CopyBuffer(env, m.pkts, m.n ? m.pkt_off[m.n] : 0));
    napi_set_named_property(env, res, "pktOff", U32Array(env, m.n ? m.pkt_off : &zero, (size_t)m.n + 1));
    napi_set_named_property(env, res, "srcIp", U32Array(env, m.src_ip, m.n));
    napi_set_named_property(env, res, "srcPort", U32Array(env, m.src_port, m.n));
    return res;
}
static bool U32Of(napi_env env, napi_value v, size_t n, const uint32_t** p) {
    napi_typedarray_type tt; size_t len; void* d; napi_value ab; size_t bo;
    if (napi_get_typedarray_info(env, v, &tt, &len, &d, &ab, &bo) != napi_ok || tt != napi_uint32_array || len != n) return false;
    *p = (const uint32_t*)d;
    return true;
}
static napi_value BackendRelay(napi_env env, napi_callback_info info) {
    size_t argc = 7; napi_value argv[7];
    NAPI_OK(napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr));
    bb_backend* b = BackendOf(env, argv[0]); if (!b) return Throw(env, BB_ERR_ARG);
    void* pk; size_t pklen; NAPI_OK(napi_get_buffer_info(env, argv[1], &pk, &pklen));
    void* up; size_t uplen; NAPI_OK(napi_get_buffer_info(env, argv[3], &up, &uplen));
    const uint32_t *qo, *uo, *ip, *port; size_t qn, un;
    if (!check_off(env, argv[2], pklen, &qo, &qn) || !check_off(env, argv[4], uplen, &uo, &un) || qn != un ||
        !U32Of(env, argv[5], qn - 1, &ip) || !U32Of(env, argv[6], qn - 1, &port)) return Throw(env, BB_ERR_ARG);
    const uint8_t* out = nullptr; size_t out_len = 0;
    int rc = bb_backend_relay(b, (const uint8_t*)pk, qo, (const uint8_t*)up, uo, ip, port, (uint32_t)(qn - 1), &out, &out_len);
    if (rc == BB_ERR_ARG) return Throw(env, rc);              // a failed batch is counted (backendStats), not thrown
    return CopyBuffer(env, out, out_len);
}
static napi_value BackendStats(napi_env env, napi_callback_info info) {
    size_t argc = 1; napi_value argv[1];
    NAPI_OK(napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr));
    bb_backend* b = BackendOf(env, argv[0]); if (!b) return Throw(env, BB_ERR_ARG);
    void* p; napi_value ab, t;
    NAPI_OK(napi_create_arraybuffer(env, 10 * 8, &p, &ab)); NAPI_OK(napi_create_typedarray(env, napi_biguint64_array, 10, ab, 0, &t));
    for (int i = 0; i < 10; i++) ((uint64_t*)p)[i] = bb_backend_stat(b, i);
    return t;
}
static napi_value BackendSetQueryLog(napi_env env, napi_callback_info info) {
    size_t argc = 2; napi_value argv[2];
    NAPI_OK(napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr));
    bb_backend* b = BackendOf(env, argv[0]); if (!b) return Throw(env, BB_ERR_ARG);
    bool on = false; NAPI_OK(napi_get_value_bool(env, argv[1], &on));
    const int rc = bb_query_log_backend_enable(b, on ? 1 : 0);
    return rc == BB_OK ? nullptr : Throw(env, rc);
}
static napi_value BackendQueryLog(napi_env env, napi_callback_info info) {
    size_t argc = 2; napi_value argv[2];
    NAPI_OK(napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr));
    bb_backend* b = BackendOf(env, argv[0]); if (!b) return Throw(env, BB_ERR_ARG);
    uint32_t which = 0; NAPI_OK(napi_get_value_uint32(env, argv[1], &which));
    bb_query_log_records r;
    const int rc = bb_query_log_backend(b, (int)std::min(which, 2u), &r);
    return rc == BB_OK ? QueryLogObject(env, r) : Throw(env, rc);
}
static napi_value BackendDestroy(napi_env env, napi_callback_info info) {
    size_t argc = 1; napi_value argv[1];
    NAPI_OK(napi_get_cb_info(env, info, &argc, argv, nullptr, nullptr));
    void* p; NAPI_OK(napi_get_value_external(env, argv[0], &p));
    bb_backend_destroy(((BackendRef*)p)->b);
    ((BackendRef*)p)->b = nullptr;                            // the finalizer then frees only the reference
    return nullptr;
}

static napi_value Init(napi_env env, napi_value exports) {
    napi_property_descriptor d[] = {
        { "zoneBuild", nullptr, ZoneBuild, nullptr, nullptr, nullptr, napi_default, nullptr },
        { "engineCreate", nullptr, EngineCreate, nullptr, nullptr, nullptr, napi_default, nullptr },
        { "engineSwapZone", nullptr, EngineSwapZone, nullptr, nullptr, nullptr, napi_default, nullptr },
        { "zoneApply", nullptr, ZoneApply, nullptr, nullptr, nullptr, napi_default, nullptr },
        { "engineApplyUpdate", nullptr, EngineApplyUpdate, nullptr, nullptr, nullptr, napi_default, nullptr },
        { "engineSetRecursionFilter", nullptr, EngineSetRecursionFilter, nullptr, nullptr, nullptr, napi_default, nullptr },
        { "resolveBatch", nullptr, ResolveBatch, nullptr, nullptr, nullptr, napi_default, nullptr },
        { "relayBatch", nullptr, RelayBatch, nullptr, nullptr, nullptr, napi_default, nullptr },
        { "logBatch", nullptr, LogBatch, nullptr, nullptr, nullptr, napi_default, nullptr },
        { "engineSetRecursionUpstreams", nullptr, EngineSetRecursionUpstreams, nullptr, nullptr, nullptr, napi_default, nullptr },
        { "forwardBatch", nullptr, ForwardBatch, nullptr, nullptr, nullptr, napi_default, nullptr },
        { "matchUpstreams", nullptr, MatchUpstreams, nullptr, nullptr, nullptr, napi_default, nullptr },
        { "tcpHubCreate", nullptr, TcpHubCreate, nullptr, nullptr, nullptr, napi_default, nullptr },
        { "tcpHubOpen", nullptr, TcpHubOpen, nullptr, nullptr, nullptr, napi_default, nullptr },
        { "tcpHubFeed", nullptr, TcpHubFeed, nullptr, nullptr, nullptr, napi_default, nullptr },
        { "tcpHubEof", nullptr, TcpHubEof, nullptr, nullptr, nullptr, napi_default, nullptr },
        { "tcpHubFlush", nullptr, TcpHubFlush, nullptr, nullptr, nullptr, napi_default, nullptr },
        { "tcpHubOutput", nullptr, TcpHubOutput, nullptr, nullptr, nullptr, napi_default, nullptr },
        { "tcpHubConsume", nullptr, TcpHubConsume, nullptr, nullptr, nullptr, napi_default, nullptr },
        { "tcpHubClose", nullptr, TcpHubClose, nullptr, nullptr, nullptr, napi_default, nullptr },
        { "tcpHubRelay", nullptr, TcpHubRelay, nullptr, nullptr, nullptr, napi_default, nullptr },
        { "tcpHubStats", nullptr, TcpHubStats, nullptr, nullptr, nullptr, napi_default, nullptr },
        { "tcpHubSetQueryLog", nullptr, TcpHubSetQueryLog, nullptr, nullptr, nullptr, napi_default, nullptr },
        { "tcpHubQueryLog", nullptr, TcpHubQueryLog, nullptr, nullptr, nullptr, napi_default, nullptr },
        { "backendCreate", nullptr, BackendCreate, nullptr, nullptr, nullptr, napi_default, nullptr },
        { "backendFeed", nullptr, BackendFeed, nullptr, nullptr, nullptr, napi_default, nullptr },
        { "backendRelay", nullptr, BackendRelay, nullptr, nullptr, nullptr, napi_default, nullptr },
        { "backendStats", nullptr, BackendStats, nullptr, nullptr, nullptr, napi_default, nullptr },
        { "backendSetQueryLog", nullptr, BackendSetQueryLog, nullptr, nullptr, nullptr, napi_default, nullptr },
        { "backendQueryLog", nullptr, BackendQueryLog, nullptr, nullptr, nullptr, napi_default, nullptr },
        { "backendDestroy", nullptr, BackendDestroy, nullptr, nullptr, nullptr, napi_default, nullptr },
    };
    napi_define_properties(env, exports, sizeof d / sizeof d[0], d);
    return exports;
}
NAPI_MODULE(NODE_GYP_MODULE_NAME, Init)
