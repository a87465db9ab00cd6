// CPU emulation of the resolve kernel: the SAME per-query device source (binder_b200/csrc/resolve_device.cuh:
// decode, lookup, resolve()/resolvePtr() decisions, sizing, both response writers) compiled for the host through
// tests/native/cuda_shim.h, driven tile by tile the way bbk::resolve_kernel drives it (staging into an emulated
// shared memory, CTA scan, placement, staged + swizzled or direct emit, flush).  The tile driver below is a
// sequential restatement of the kernel body; the per-query functions are the device code itself.  Lets kernel logic
// be checked against the oracle without a GPU (tests/test_host_emulation.py).  Test infrastructure, not product.
#include "cuda_shim.h"
#include "../../binder_b200/csrc/zone_image.h"
#include "../../include/binder_b200.h"
namespace bbk { thread_local unsigned long long bb_emu_lean_count = 0, bb_emu_general_count = 0; }
#include "../../binder_b200/csrc/resolve_device.cuh"

#include <vector>
#include <cstdio>
#include <cstdlib>

thread_local uint8_t* bb_emu_smem = nullptr;
// what the copy-job machinery saw so far: big tiles, job-mode responses, responses whose jobs did not fit the list, jobs
// with a masked tail, emit rounds
static thread_local unsigned long long g_job_stats[5];
extern "C" void bb_emu_job_stats(unsigned long long* out, int reset) { for (int i = 0; i < 5; i++) { out[i] = g_job_stats[i]; if (reset) g_job_stats[i] = 0; } }
extern "C" const bb::ZoneImage* bb_zone_image(const bb_zone* z);

namespace {
using namespace bbk;
constexpr size_t OFF_IN = 16;                              // s_in  [S_IN + 32]; never 0: Res::sp == 0 means "not staged"
constexpr size_t OFF_OUT = 9216;                           // s_out [S_OUT], 1024-aligned like the kernel's
constexpr size_t OFF_SFX = OFF_OUT + ((S_OUT + 1023) / 1024) * 1024;
constexpr size_t OFF_OPT = OFF_SFX + 256 + 64;              // the OPT RR's bytes (a copy-job source)
constexpr size_t SMEM_BYTES = OFF_OPT + 16 + 64;
static_assert(OFF_OUT >= OFF_IN + S_IN + 32 && OFF_OUT % 1024 == 0, "layout");
}

static int emu_resolve_image(const bb::ZoneImage* img, const bb::EngineConst& C,
                             const uint8_t* pkts, const uint32_t* pkt_off, uint32_t n, uint64_t seed, uint32_t qidx_base,
                             int ordered, int tcp, uint8_t* out, uint32_t out_cap, uint32_t* out_off, uint16_t* out_len,
                             uint8_t* status, uint32_t* miss_idx, uint32_t* n_miss, const uint32_t* qidx_map);

extern "C" int bb_emu_resolve_batch(const bb_zone* zone, const char* dns_domain, int recursion,
                                    const char* rf_region, const char* const* rf_dcs, uint32_t rf_n, int rf_ptr,
                                    const uint8_t* pkts, const uint32_t* pkt_off, uint32_t n, uint64_t seed, uint32_t qidx_base,
                                    int ordered, int tcp, uint8_t* out, uint32_t out_cap, uint32_t* out_off, uint16_t* out_len,
                                    uint8_t* status, uint32_t* miss_idx, uint32_t* n_miss, const uint32_t* qidx_map) {
    bb::EngineConst C;
    if (!bb::make_engine_const(dns_domain, recursion != 0, C)) return BB_ERR_DOMAIN;
    if (rf_region && !bb::set_recursion_filter_const(C, rf_region, rf_dcs, rf_n, rf_ptr != 0)) return BB_ERR_ARG;
    return emu_resolve_image(zone ? bb_zone_image(zone) : nullptr, C, pkts, pkt_off, n, seed, qidx_base, ordered, tcp, out, out_cap, out_off, out_len,
                             status, miss_idx, n_miss, qidx_map);
}

static int emu_resolve_image(const bb::ZoneImage* img, const bb::EngineConst& C,
                             const uint8_t* pkts, const uint32_t* pkt_off, uint32_t n, uint64_t seed, uint32_t qidx_base,
                             int ordered, int tcp, uint8_t* out, uint32_t out_cap, uint32_t* out_off, uint16_t* out_len,
                             uint8_t* status, uint32_t* miss_idx, uint32_t* n_miss, const uint32_t* qidx_map) {
    static thread_local std::vector<uint8_t> smem(SMEM_BYTES + 1024);
    bb_emu_smem = (uint8_t*)(((uintptr_t)smem.data() + 1023) & ~(uintptr_t)1023);     // offsets == emulated shared addresses
    Params P; memset(&P, 0, sizeof P);
    P.pkts = pkts; P.pkt_off = pkt_off; P.n = n; P.seed = seed; P.qidx_base = qidx_base;
    P.out = out; P.out_cap = out_cap; P.out_off = out_off; P.out_len = out_len; P.status = status; P.miss_idx = miss_idx;
    P.table = img ? img->slots : nullptr; P.mask = img ? img->nslots - 1 : 0; P.arena = img ? img->arena : nullptr;
    P.ready = img && img->ready; P.eng = &C; P.suffix_len = C.suffix_len; P.soa_len = C.soa_len; P.recursion = C.recursion; P.lean_ok = C.lean_ok;
    P.nranks = 1; P.tcp = tcp ? 1u : 0u;
    (void)ordered;                                          // one tile at a time: arrival order IS query order here
    uint8_t* s_in = bb_emu_smem + OFF_IN; uint8_t* s_out = bb_emu_smem + OFF_OUT; uint8_t* s_sfx = bb_emu_smem + OFF_SFX;
    memcpy(s_sfx, C.wire_tail, 256);
    uint64_t gbase = 0; uint32_t mbase = 0;
    for (uint32_t q0 = 0; q0 < n; q0 += T) {
        const uint32_t nq = std::min<uint32_t>(T, n - q0);
        blockIdx.x = q0 / T;
        const uint32_t* s_off = pkt_off + q0;
        const uint32_t b0 = s_off[0], b1 = s_off[nq], a0 = b0 & ~15u;
        const bool staged = b1 >= b0 && b1 - a0 <= (uint32_t)S_IN;
        if (staged) memcpy(s_in, pkts + a0, ((b1 - a0 + 15) >> 4) << 4);            // the batch container is padded for this
        Res r[T]; uint32_t qidx[T];
        uint32_t tile_bytes = 0, tile_miss = 0, my_o[T], my_m[T];
        for (uint32_t t = 0; t < nq; t++) {
            threadIdx.x = t;
            r[t].status = ST_DROPPED; r[t].rlen = 0; r[t].rk = RK_NONE; r[t].trunc = 0; r[t].sp = 0; r[t].ntask = 0;
            qidx[t] = qidx_map ? qidx_map[q0 + t] : qidx_base + q0 + t;     // routed batches carry their ingress index
            const uint32_t o0 = s_off[t], o1 = s_off[t + 1];
            if (o1 >= o0 && o1 - o0 <= 65535u) {
                r[t].p = staged ? s_in + (o0 - a0) : pkts + o0;
                r[t].sp = staged ? (uint32_t)(OFF_IN + (o0 - a0)) : 0u;
                resolve_query(P, r[t], o1 - o0, qidx[t], (uint32_t)OFF_SFX);
            }
            my_o[t] = tile_bytes; my_m[t] = tile_miss;
            tile_bytes += r[t].rlen; tile_miss += r[t].status == ST_MISS;
        }
        if (gbase + tile_bytes > out_cap) return BB_ERR_CAPACITY;
        bool odd = false;
        for (uint32_t t = 0; t < nq; t++) {
            out_off[q0 + t] = (uint32_t)(gbase + my_o[t]); out_len[q0 + t] = r[t].rlen; status[q0 + t] = r[t].status;
            if (r[t].status == ST_MISS) miss_idx[mbase + my_m[t]] = q0 + t;
            odd |= r[t].rlen && (!(r[t].sp && !r[t].trunc) || r[t].rlen > (uint32_t)MAXRESP);
        }
        if (odd) {
            for (uint32_t t = 0; t < nq; t++) {
                if (!r[t].rlen) continue;
                threadIdx.x = t;
                if (!(r[t].sp && !r[t].trunc)) emit_response(P, r[t], out + gbase + my_o[t], qidx[t]);
                else { WrT<2> w; w.begin_global(out, (uint32_t)(gbase + my_o[t])); emit_fast(P, r[t], w, qidx[t]); }
            }
        } else if (tile_bytes) {
            // the service variant's emit: one round when the tile fits the window; else rounds over the responses that START in
            // each window, the job-mode service answers as copy jobs in ONE list in tile-offset order (a thread's jobs at the
            // exclusive prefix of the job counts), each round running its own contiguous run of the list
            const bool big = tile_bytes > (uint32_t)WIN;
            static thread_local std::vector<Task> tl; static thread_local std::vector<uint8_t> jobs; static thread_local std::vector<uint32_t> tbase;
            tl.resize(TASKCAP); jobs.assign(nq, 0); tbase.assign(nq + 1, 0);
            const uint32_t opt_words[4] = { 0x04290000u, 0x000000B0u, 0u, 0u };
            memcpy(bb_emu_smem + OFF_OPT, opt_words, 16);
            uint32_t tv = 0;
            if (big) {
                for (uint32_t t = 0; t < nq; t++) {
                    uint32_t cnt = 0;
                    if (r[t].rlen && r[t].ntask) {
                        threadIdx.x = t; TaskCount tc = { 0 }; plan_service(P, r[t], qidx[t], 0, 0, tc); cnt = tc.n;
                        if (r[t].ntask >= 2 && r[t].ntask - 2 != cnt) return BB_ERR_ARG;          // the build-time job count must be the walk's
                    }
                    tbase[t + 1] = tbase[t] + cnt;
                }
                tv = std::min<uint32_t>(tbase[nq], TASKCAP);
                g_job_stats[0]++;
                for (uint32_t t = 0; t < nq; t++) {
                    const uint32_t cnt = tbase[t + 1] - tbase[t];
                    if (!cnt) continue;
                    threadIdx.x = t;
                    if (tbase[t] + cnt <= (uint32_t)TASKCAP) { TaskFill f = { tl.data() + tbase[t] }; plan_service(P, r[t], qidx[t], my_o[t], (uint32_t)OFF_OPT, f); jobs[t] = 1; g_job_stats[1]++;
                        for (uint32_t i = tbase[t]; i < tbase[t] + cnt; i++) g_job_stats[3] += task_exact(tl[i]); }
                    else { tv = std::min(tv, tbase[t]); g_job_stats[2]++; }
                }
            }
            const uint32_t nr = big ? (tile_bytes + WIN - 1) / WIN : 1u;
            for (uint32_t k = 0; k < nr; k++) {
                uint32_t x0 = 0xFFFFFFFFu, x1 = tile_bytes, t0 = 0xFFFFFFFFu, t1 = tv;
                for (uint32_t t = 0; t < nq; t++) if (r[t].rlen) {
                    const uint32_t kr = big ? my_o[t] / WIN : 0u;
                    if (kr == k) { x0 = std::min(x0, my_o[t]); t0 = std::min(t0, tbase[t]); }
                    else if (kr > k && my_o[t] < x1) { x1 = my_o[t]; t1 = std::min(tbase[t], tv); }
                }
                if (x0 == 0xFFFFFFFFu) continue;
                g_job_stats[4] += big;
                t0 = std::min(t0, tv);
                const uint32_t shift = (uint32_t)((gbase + x0) & 15), delta = shift - x0;
                if (shift + (x1 - x0) > (uint32_t)S_OUT) return BB_ERR_CAPACITY;                        // cannot happen: WIN + MAXRESP <= CAPW
                if (big) memset(s_out, 0, S_OUT);                                                         // pieces are OR-ed into a zeroed buffer
                for (uint32_t t = 0; t < nq; t++) {
                    if (!r[t].rlen || (big ? my_o[t] / WIN : 0u) != k) continue;
                    threadIdx.x = t;
                    if (big) { WrT<4> w; w.begin((uint32_t)OFF_OUT, delta + my_o[t]); if (jobs[t]) { emit_head_w(r[t], w); w.end(); } else emit_fast(P, r[t], w, qidx[t]); }
                    else { WrT<1> w; w.begin((uint32_t)OFF_OUT, delta + my_o[t]); emit_fast(P, r[t], w, qidx[t]); }
                }
                if (big) for (uint32_t t = 0; t < (uint32_t)T; t++) run_tasks(P, tl.data(), t0, t1, t, (uint32_t)OFF_OUT + delta);
                if (big) for (uint32_t x = x0; x < x1; x++) out[gbase + x] = s_out[delta + x];         // the flush (linear buffer)
                else for (uint32_t x = x0; x < x1; x++) out[gbase + x] = s_out[swz(delta + x)];         // the flush (swizzled buffer)
            }
        }
        gbase += tile_bytes; mbase += tile_miss;
    }
    out_off[n] = (uint32_t)gbase;
    *n_miss = mbase;
    return BB_OK;
}

// ---- the CPU baseline "same table, same algorithm" (SURVEY.md section 8d): the word-wise device code over the SAME zone
// image (the cuckoo table and the arena the GPU probes), on `nthreads` host threads, each taking a contiguous run of whole
// tiles with its own output buffers.  `image` = the bb::ZoneImage of a built zone (bb_zone_image()).  Writes the best
// wall-clock seconds of `repeat` passes; returns BB_OK, or the first error of any thread.
#include <chrono>
#include <condition_variable>
#include <mutex>
#include <thread>
extern "C" int bb_emu_timed_resolve(const void* image, const char* dns_domain, int recursion, const uint8_t* pkts, const uint32_t* pkt_off,
                                    uint32_t n, uint64_t seed, uint32_t nthreads, uint32_t repeat, uint32_t resp_cap_per_query,
                                    double* best_secs, uint64_t* total_bytes, uint64_t* total_miss) {
    bb::EngineConst C;
    if (!image || !nthreads || !repeat || !bb::make_engine_const(dns_domain, recursion != 0, C)) return BB_ERR_ARG;
    const bb::ZoneImage* img = (const bb::ZoneImage*)image;
    const uint32_t ntiles = (n + T - 1) / T;
    if (nthreads > ntiles) nthreads = ntiles ? ntiles : 1;
    // `skew`: the slices' buffers are page-aligned allocations of equal size; started at the same offset the threads would
    // walk them in lockstep on identical cache sets
    struct Slice { uint32_t q0, q1; size_t skew; std::vector<uint8_t> out, status; std::vector<uint32_t> off, miss; std::vector<uint16_t> len; uint32_t nmiss = 0; int rc = 0; };
    std::vector<Slice> sl(nthreads);
    for (uint32_t t = 0; t < nthreads; t++) {
        const uint32_t t0 = (uint32_t)((uint64_t)ntiles * t / nthreads), t1 = (uint32_t)((uint64_t)ntiles * (t + 1) / nthreads);
        Slice& s = sl[t]; s.q0 = std::min(n, t0 * T); s.q1 = std::min(n, t1 * T);
        const uint32_t m = s.q1 - s.q0;
        s.skew = (size_t)t * 4160;
        s.out.assign((size_t)m * resp_cap_per_query + 64 + s.skew, 0); s.status.assign(m + 1, 0); s.off.assign(m + 1, 0); s.miss.assign(m + 1, 0); s.len.assign(m + 1, 0);
    }
    // the workers live for the whole call and meet at a barrier per pass; pass 0 is a warm-up (their stacks, thread-local
    // buffers and output pages are touched there), passes 1..repeat are timed from the main thread
    struct Barrier {
        std::mutex m; std::condition_variable cv; uint32_t n, waiting = 0, gen = 0;
        void wait() { std::unique_lock<std::mutex> l(m); const uint32_t g = gen; if (++waiting == n) { waiting = 0; ++gen; cv.notify_all(); } else cv.wait(l, [&] { return gen != g; }); }
    } bar; bar.n = nthreads + 1;
    std::vector<std::thread> th;
    for (uint32_t t = 0; t < nthreads; t++) th.emplace_back([&, t] {
        Slice& s = sl[t];
        const uint32_t m = s.q1 - s.q0;
        for (uint32_t rep = 0; rep <= repeat; rep++) {
            bar.wait();
            // the slice as a batch of its own: offsets are absolute in `pkts`, so the packets pointer stays and the offsets shift
            if (m && !s.rc)
                s.rc = emu_resolve_image(img, C, pkts, pkt_off + s.q0, m, seed, s.q0, 1, 0, s.out.data() + s.skew, (uint32_t)std::min<size_t>(s.out.size() - 64 - s.skew, 0xFFFFFF00u),
                                         s.off.data(), s.len.data(), s.status.data(), s.miss.data(), &s.nmiss, nullptr);
            bar.wait();
        }
    });
    double best = 1e30;
    for (uint32_t rep = 0; rep <= repeat; rep++) {
        const auto a = std::chrono::steady_clock::now();
        bar.wait(); bar.wait();
        const double d = std::chrono::duration<double>(std::chrono::steady_clock::now() - a).count();
        if (rep && d < best) best = d;
    }
    for (auto& x : th) x.join();
    uint64_t tb = 0, tm = 0;
    for (auto& s : sl) { if (s.rc) return s.rc; tb += s.off[s.q1 - s.q0]; tm += s.nmiss; }
    *best_secs = best; *total_bytes = tb; *total_miss = tm;
    return BB_OK;
}

// which front end settled the queries so far: [0] lean_query, [1] complete decoder + generic path
extern "C" void bb_emu_path_counts(unsigned long long* out, int reset) {
    out[0] = bbk::bb_emu_lean_count; out[1] = bbk::bb_emu_general_count;
    if (reset) bbk::bb_emu_lean_count = bbk::bb_emu_general_count = 0;
}

// Where a key lives in a built zone's table (tests/test_table_probe.py proves the states it crafts with this): the table
// mask, both hashes, the slot that holds the key (UINT32_MAX: neither of its two slots does) and whether the key's FIRST
// position carries SLOT_DISPLACED.  `key` is the canonical form (forward: wire labels; reverse: the address string).  The
// bytes are compared here, on the image itself, not through the builder's lookup.  Returns 1 when the key is present.
extern "C" int bb_emu_slot_of(const bb_zone* zone, uint32_t ns, const uint8_t* key, uint32_t len, uint32_t* mask, uint32_t* slot,
                              int* first_displaced, uint32_t* h_out, uint32_t* h2_out) {
    const bb::ZoneImage* img = zone ? bb_zone_image(zone) : nullptr;
    if (!img || !img->slots) return -1;
    uint32_t h2;
    const uint32_t h = bb::hash_key2(ns, key, len, &h2), m = img->nslots - 1;
    *mask = m; *h_out = h; *h2_out = h2; *slot = 0xFFFFFFFFu;
    *first_displaced = (img->slots[bb::slot1_of(h, m)].flags & bb::SLOT_DISPLACED) ? 1 : 0;
    for (uint32_t i : { bb::slot1_of(h, m), bb::slot2_of(h, h2, m) }) {
        const bb::Slot& s = img->slots[i];
        if (s.kind == bb::K_EMPTY || s.ns != ns) continue;
        const uint8_t* kb = nullptr;
        if (s.klen == bb::KLEN_OVERFLOW) {
            uint32_t off, l;
            memcpy(&off, s.key, 4); memcpy(&l, s.key + 4, 4);
            if (l == len && off + (uint64_t)len <= img->arena_len) kb = img->arena + off;
        } else if (s.klen == len) kb = s.key;
        if (kb && memcmp(kb, key, len) == 0) { *slot = i; return 1; }
    }
    return 0;
}

// Route mode (the ingress half of the sharded path, route_push_kernel's per-query step): which rank owns each
// query's lookup key; queries that need no lookup stay on `rank`.
extern "C" int bb_emu_route_batch(const char* dns_domain, int recursion, const uint8_t* pkts, const uint32_t* pkt_off, uint32_t n,
                                  uint32_t nranks, uint32_t rank, uint8_t* owner) {
    static thread_local std::vector<uint8_t> smem(SMEM_BYTES + 1024);
    bb_emu_smem = (uint8_t*)(((uintptr_t)smem.data() + 1023) & ~(uintptr_t)1023);
    bb::EngineConst C;
    if (!bb::make_engine_const(dns_domain, recursion != 0, C)) return BB_ERR_DOMAIN;
    Params P; memset(&P, 0, sizeof P);
    P.pkts = pkts; P.pkt_off = pkt_off; P.n = n; P.eng = &C; P.ready = 1;
    P.suffix_len = C.suffix_len; P.soa_len = C.soa_len; P.recursion = C.recursion; P.lean_ok = C.lean_ok;
    P.route = 1; P.nranks = nranks; P.rank = rank;
    uint8_t* s_in = bb_emu_smem + OFF_IN;
    memcpy(bb_emu_smem + OFF_SFX, C.wire_tail, 256);
    for (uint32_t q0 = 0; q0 < n; q0 += T) {
        const uint32_t nq = std::min<uint32_t>(T, n - q0);
        const uint32_t* s_off = pkt_off + q0;
        const uint32_t b0 = s_off[0], b1 = s_off[nq], a0 = b0 & ~15u;
        const bool staged = b1 >= b0 && b1 - a0 <= (uint32_t)S_IN;
        if (staged) memcpy(s_in, pkts + a0, ((b1 - a0 + 15) >> 4) << 4);
        for (uint32_t t = 0; t < nq; t++) {
            Res r; r.owner = (uint8_t)rank; r.sp = 0; r.p = nullptr;
            const uint32_t o0 = s_off[t], o1 = s_off[t + 1];
            if (o1 >= o0 && o1 - o0 <= 65535u) {
                r.p = staged ? s_in + (o0 - a0) : pkts + o0;
                r.sp = staged ? (uint32_t)(OFF_IN + (o0 - a0)) : 0u;
                resolve_query(P, r, o1 - o0, 0, (uint32_t)OFF_SFX);
                if (r.owner >= nranks) r.owner = (uint8_t)rank;
            }
            owner[q0 + t] = r.owner;
        }
    }
    return BB_OK;
}
