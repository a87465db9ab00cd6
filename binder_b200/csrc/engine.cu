// binder_b200 engine: the CUDA resolve kernel for sm_100a and the host side of the C ABI.
//
// One kernel does the whole of binder's per-query path for a batch of raw DNS packets:
//   mname decode                      -> decode()                 (call site lib/server.js:443-446,471)
//   onQuery type dispatch             -> resolve_query()          (lib/server.js:491-506)
//   resolve / resolvePtr              -> resolve_forward/_ptr()   (lib/server.js:67-134,136-429)
//   zkCache.lookup / reverseLookup    -> probe()                  (lib/zk.js:62-67)
//   shuffle                           -> make_perm()/perm_at()    (lib/server.js:40-53)
//   mname encode + respond            -> emit_response()          (lib/server.js:130,286,299,310,398-402,413-414,427)
//   miss hand-off to recursion        -> compacted miss_idx[]     (lib/server.js:110-113,222-225)
//
// Data movement (HBM-bound integer/byte work, no tensor cores):
//   * a CTA owns a tile of 128 consecutive queries; their packed bytes are one contiguous
//     range of the input, staged into shared memory with coalesced 16-byte loads;
//   * each thread parses its packet from shared memory, hashes the normalised name and
//     probes the zone table in HBM (one 32-byte slot = one sector per host record);
//   * response sizes are scanned in the CTA, tile bases come from a single-pass decoupled
//     look-back across CTAs (so output is packed, in query order, in ONE kernel);
//   * responses are assembled in shared memory and flushed with 16-byte coalesced stores.
#include "zone_image.h"
#include "../../include/binder_b200.h"

#include <cuda_runtime.h>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

extern "C" const bb::ZoneImage* bb_zone_image(const bb_zone* z);
extern "C" int bb_zone_pending(const bb_zone* z, const uint32_t** slots, uint32_t* n_slots, uint64_t* arena_from, int* relaid);
extern "C" void bb_zone_mark_synced(bb_zone* z);
extern "C" uint64_t bb_zone_sync_gen(const bb_zone* z);

#include "resolve_device.cuh"

namespace bbk {
// ---- the kernel ------------------------------------------------------------------------------
__device__ __forceinline__ uint64_t warp_sum64(uint64_t v) {
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// ---- bulk asynchronous copies (the TMA unit's 1-D form) and the mbarrier they complete on ------------------------
// A tile's packets are ONE contiguous, 16-byte aligned byte range of the batch: one thread hands the range to the
// copy engine (cp.async.bulk global -> shared), the engine counts the bytes in on an mbarrier, everybody waits on the
// barrier's phase.  No thread issues loads or stores for the staging and no register holds packet bytes in flight.
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(bar), "r"(count) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");       // visible to the async proxy before the copy is issued
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {      // bytes: multiple of 16
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 :: "r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}
// wait for phase `parity` of the barrier; a bounded spin (a copy that never lands is a bug: trap instead of hanging the device)
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    for (uint32_t spin = 0;; spin++) {
        uint32_t ok;
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                     : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
        if (ok) return;
        if (spin > (1u << 24)) __trap();
    }
}
// shared -> global, issued by one thread after the writers' generic-proxy stores were fenced and the block synchronised
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void bulk_s2g(void* dst, uint32_t src, uint32_t bytes) {                            // bytes: multiple of 16
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" :: "l"(dst), "r"(src), "r"(bytes) : "memory");
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
}
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }

// 6 tiles (768 threads) resident per SM: 80 registers (96 for the service variant).  On sm_90a the 64-register cap of
// 8 tiles spills ~600 bytes per thread, and 6 measured faster on an H100 on configs 2 and 3 (DESIGN.md section 5).
#ifndef BB_MIN_BLOCKS
#define BB_MIN_BLOCKS 6
#endif
// ORDERED: responses packed in query order (tile bases from a decoupled look-back; a tile waits
// for its predecessors' sizes).  !ORDERED ("arrival" packing): a tile claims its output range
// with one atomicAdd and never waits; response i is still out[out_off[i] .. +out_len[i]).
// MULTI: one launch over several receive regions (routed batches, grid.y = source rank): every
// per-batch pointer advances by its stride per region, sizes and shuffle indices come from device memory.
// SVC: the variant for batches of long (service) answers — copy-job lists in shared memory and emit rounds; it fits one tile per
// SM fewer, which batches of 64-byte answers would feel, so the host picks per batch (engine: the previous batch's
// mean response size).  Both variants answer every batch correctly.
template <bool ORDERED, bool MULTI, bool SVC>
__global__ void __launch_bounds__(T, SVC ? BB_MIN_BLOCKS - 1 : BB_MIN_BLOCKS) resolve_kernel(const Params P) {
    // the packets start 16 bytes in: a staged packet's shared address is never 0 (Res::sp == 0 means "not staged")
    __shared__ __align__(16) uint8_t s_inbuf[16 + S_IN + 32];
    uint8_t* const s_in = s_inbuf + 16;
    __shared__ __align__(1024) uint8_t s_out[S_OUT];         // XOR-swizzled (swz()); 1024-aligned: WrT<1> swizzles addresses
    __shared__ uint32_t s_off[T + 1];
    __shared__ uint32_t s_wsum[8];
    __shared__ uint32_t s_rstart[NROUNDS + 1];                 // big tiles: tile offset of each emit round's first response
    __shared__ uint32_t s_tstart[NROUNDS + 2];                 // big tiles: each emit round's first copy job; [NROUNDS + 1] = jobs that fit the list
    __shared__ uint32_t s_wsum2[T / 32];                       // service variant: the warps' job counts (second scan)
    __shared__ Task s_task[SVC ? TASKCAP : 1];                 // big tiles: the copy jobs, in tile-offset order
    __shared__ uint8_t s_perm[T];                              // which query of the tile each thread takes (grouped by question type)
    __shared__ uint32_t s_opt[4];                              // the OPT RR's 11 bytes, as a job source
    __shared__ unsigned long long s_prefix;
    __shared__ __align__(8) unsigned long long s_bar;        // mbarrier of the input staging copy
    __shared__ __align__(16) uint8_t s_sfx[256];            // dnsDomain as wire labels, right-aligned (EngineConst::wire_tail)
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const size_t ry = MULTI ? blockIdx.y : 0;
    const uint8_t* const r_pkts = MULTI ? P.pkts + ry * P.in_stride : P.pkts;
    const uint32_t* const r_pkt_off = MULTI ? (const uint32_t*)((const uint8_t*)P.pkt_off + ry * P.in_stride) : P.pkt_off;
    const uint32_t* const r_n_dev = (MULTI && P.n_dev) ? (const uint32_t*)((const uint8_t*)P.n_dev + ry * P.in_stride) : nullptr;
    const uint32_t* const r_qidx_map = (MULTI && P.qidx_map) ? (const uint32_t*)((const uint8_t*)P.qidx_map + ry * P.in_stride) : nullptr;
    uint8_t* const r_out = MULTI ? P.out + ry * P.out_stride : P.out;
    uint32_t* const r_out_off = MULTI ? (uint32_t*)((uint8_t*)P.out_off + ry * P.off_stride) : P.out_off;
    uint16_t* const r_out_len = MULTI ? (uint16_t*)((uint8_t*)P.out_len + ry * P.len_stride) : P.out_len;
    uint8_t* const r_status = MULTI ? P.status + ry * P.status_stride : P.status;
    uint32_t* const r_miss_idx = MULTI ? (uint32_t*)((uint8_t*)P.miss_idx + ry * P.miss_stride) : P.miss_idx;
    uint32_t* const r_totals = MULTI ? (uint32_t*)((uint8_t*)P.totals + ry * P.totals_stride) : P.totals;
    unsigned long long* const r_desc = MULTI ? (unsigned long long*)((uint8_t*)P.desc + ry * P.desc_stride) : P.desc;
    uint32_t* const r_counter = MULTI ? (uint32_t*)((uint8_t*)P.counter + ry * P.desc_stride) : P.counter;
    uint32_t* const r_qidx_out = (MULTI && P.qidx_out) ? (uint32_t*)((uint8_t*)P.qidx_out + ry * P.off_stride) : nullptr;
    uint8_t* const r_bounce = (MULTI && P.bounce) ? P.bounce + ry * P.out_stride : P.bounce;

    // Tiles are taken in blockIdx order: like CUB's single-pass scan, the look-back below relies on
    // thread blocks being dispatched in increasing blockIdx order (a block only ever waits for
    // lower-numbered blocks, which are resident or finished).
    for (int i = tid; i < 64; i += T) ((uint32_t*)s_sfx)[i] = __ldg((const uint32_t*)P.eng->wire_tail + i);
    const uint32_t tile = blockIdx.x;
    STAMP(0);
    // routed batches: size known only on the device (header: count, bytes, epoch, sender overflow flag)
    const uint32_t n = r_n_dev ? (r_n_dev[3] ? 0u : r_n_dev[0]) : P.n;
    const uint32_t ntiles = (n + T - 1) / T;
    if (tile < ntiles) {
    const uint32_t q0 = tile * T;
    const uint32_t nq = min((uint32_t)T, n - q0);

    // ---- stage this tile's packets ---------------------------------------------------------
    // Thread 0 reads the tile's first and last offset and hands the byte range to the copy engine; meanwhile every thread
    // loads its own packet's offset.  (The range is read again from s_off below: same memory, same values.)
    const uint32_t bar = (uint32_t)__cvta_generic_to_shared(&s_bar);
    if (tid == 0) {
        mbar_init(bar, 1);
        const uint32_t f0 = r_pkt_off[q0], f1 = r_pkt_off[q0 + nq], fa = f0 & ~15u;
        if (f1 >= f0 && f1 - fa <= (uint32_t)S_IN && f1 > fa) {
            const uint32_t bytes = (f1 - fa + 15) & ~15u;
            mbar_expect_tx(bar, bytes);
            bulk_g2s((uint32_t)__cvta_generic_to_shared(s_in), r_pkts + fa, bytes, bar);
        }
    }
    if (tid < (int)nq) s_off[tid] = r_pkt_off[q0 + tid];
    if (tid == 0) s_off[nq] = r_pkt_off[q0 + nq];
    __syncthreads();
    STAMP(1);
    const uint32_t b0 = s_off[0], b1 = s_off[nq];
    const uint32_t a0 = b0 & ~15u;
    const bool staged = b1 >= b0 && b1 - a0 <= S_IN;
    if (staged && b1 > a0) mbar_wait(bar, 0);                 // the bytes have landed (and are visible to every waiting thread)

    STAMP(2);
    // ---- parse + lookup + size ----------------------------------------------------------------
    // Which query this thread takes.  With arrival packing the order inside a tile is free, so the tile is partitioned by
    // question type: SRV queries (long, child-by-child answers) share warps with SRV queries and the rest with the
    // rest, instead of half of every warp idling through the other half's loops.  (Query-order packing keeps tid.)
    uint32_t qi = (uint32_t)tid;
    if (!ORDERED && staged) {
        bool srvq = false;
        if (tid < (int)nq) {
            const uint32_t o0 = s_off[tid], o1 = s_off[tid + 1];
            if (o0 >= b0 && o1 >= o0 + 17 && o1 <= b1) {                      // QTYPE sits 4 bytes (15 with a bare OPT) before the end
                const uint8_t* pk = s_in + (o0 - a0);
                const uint32_t back = pk[11] ? 15u : 4u, len = o1 - o0;
                srvq = len >= 12 + back && pk[len - back] == 0 && pk[len - back + 1] == QT_SRV;
            }
        }
        const uint32_t bal = __ballot_sync(0xffffffffu, srvq), before = __popc(bal & ((1u << lane) - 1));
        if (lane == 0) s_wsum[warp] = __popc(bal);
        __syncthreads();
        uint32_t srv_before = before, srv_total = 0;
        for (int w = 0; w < T / 32; w++) { const uint32_t x = s_wsum[w]; if (w < warp) srv_before += x; srv_total += x; }
        // the others first (in order), then the SRV queries (in order)
        const uint32_t pos = srvq ? (uint32_t)T - srv_total + srv_before : (uint32_t)tid - srv_before;
        s_perm[pos] = (uint8_t)tid;
        __syncthreads();
        qi = s_perm[tid];
    }
    Res r;
    r.status = ST_DROPPED; r.rlen = 0; r.rk = RK_NONE; r.ntask = 0;
    const uint32_t qidx = (r_qidx_map && qi < nq) ? r_qidx_map[q0 + qi] : P.qidx_base + q0 + qi;
    if (qi < nq) {
        const uint32_t o0 = s_off[qi], o1 = s_off[qi + 1];
        // a packet must lie inside its tile's byte range [b0, b1] (the host checked the tile boundaries against the
        // batch's size): offsets that run backwards or jump out are dropped, never dereferenced
        if (o0 >= b0 && o1 >= o0 && o1 <= b1 && o1 - o0 <= 65535u) {
            r.p = staged ? s_in + (o0 - a0) : r_pkts + o0;
            r.sp = staged ? (uint32_t)__cvta_generic_to_shared(s_in) + (o0 - a0) : 0u;
            resolve_query(P, r, o1 - o0, qidx, (uint32_t)__cvta_generic_to_shared(s_sfx));
        }
    }
    const uint32_t my_len = r.rlen;
    const uint32_t my_miss = (qi < nq && r.status == ST_MISS) ? 1u : 0u;
    // service variant: how many copy jobs this response becomes (its jobs go to the exclusive prefix of these counts)
    uint32_t my_cnt = 0;
    if (SVC && my_len && r.ntask) {
        if (r.ntask >= 2) my_cnt = r.ntask - 2;          // whole answer: the count is a build-time sum
        else { TaskCount tc = { 0 }; plan_service(P, r, qidx, 0, 0, tc); my_cnt = tc.n; }
    }

    STAMP(6);
    // ---- CTA scan of (bytes, misses) ------------------------------------------------------------
    uint32_t v = my_len | (my_miss << 24);     // 128 x 1232 < 2^24
    uint32_t inc = v, inc2 = my_cnt;
    for (int o = 1; o < 32; o <<= 1) {
        uint32_t t = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += t;
        if (SVC) { uint32_t t2 = __shfl_up_sync(0xffffffffu, inc2, o); if (lane >= o) inc2 += t2; }
    }
    if (lane == 31) { s_wsum[warp] = inc; if (SVC) s_wsum2[warp] = inc2; }
    __syncthreads();
    uint32_t wbase = 0, tot = 0, tbase = inc2 - my_cnt, ttot = 0;
    for (int w = 0; w < T / 32; w++) { uint32_t x = s_wsum[w]; if (w < warp) wbase += x; tot += x; }
    if (SVC) for (int w = 0; w < T / 32; w++) { uint32_t x = s_wsum2[w]; if (w < warp) tbase += x; ttot += x; }
    const uint32_t excl = wbase + inc - v;
    const uint32_t my_o = excl & 0xFFFFFF, my_mrank = excl >> 24;
    const uint32_t tile_bytes = tot & 0xFFFFFF, tile_miss = tot >> 24;

    STAMP(7);
    // ---- where this tile's responses (and misses) go ------------------------------------------
    if (!ORDERED) {
        if (tid == 0)                                    // one claim per tile: bytes | misses << 40
            s_prefix = atomicAdd(r_desc + P.ntiles_cap, (unsigned long long)tile_bytes | ((unsigned long long)tile_miss << D_MISS_SHIFT));
    } else
    if (warp == 0) {
        volatile unsigned long long* D = r_desc;
        const uint64_t agg = (uint64_t)tile_bytes | ((uint64_t)tile_miss << D_MISS_SHIFT);
        uint64_t ex = 0;
        if (tile == 0) { if (lane == 0) D[0] = D_FLAG_P | agg; }
        else {
            if (lane == 0) D[tile] = D_FLAG_A | agg;
            int base = (int)tile - 1;
            for (;;) {                                   // window of 128 predecessors, 4 independent loads per lane
                uint64_t d[4];
                bool ready;
                do {
                    ready = true;
#pragma unroll
                    for (int k = 0; k < 4; k++) {
                        const int idx = base - lane - 32 * k;
                        d[k] = idx >= 0 ? D[idx] : D_FLAG_P;
                        ready &= (d[k] >> 62) != 0;
                    }
                } while (__any_sync(0xffffffffu, !ready));
                uint32_t mypos = 0xFFFFFFFFu;            // distance of the nearest predecessor with an inclusive prefix
#pragma unroll
                for (int k = 3; k >= 0; k--) if ((d[k] >> 62) == 2) mypos = (uint32_t)(lane + 32 * k);
                uint32_t minpos = mypos;
                for (int o = 16; o; o >>= 1) minpos = min(minpos, __shfl_xor_sync(0xffffffffu, minpos, o));
                uint64_t part = 0;
#pragma unroll
                for (int k = 0; k < 4; k++) if ((uint32_t)(lane + 32 * k) <= minpos) part += d[k] & D_VAL;
                ex += warp_sum64(part);
                if (minpos != 0xFFFFFFFFu) break;
                base -= 128;
            }
            if (lane == 0) D[tile] = D_FLAG_P | (ex + agg);
        }
        if (lane == 0) s_prefix = ex;
    }
    __syncthreads();
    STAMP(8);
    const uint64_t ex = s_prefix;
    const uint64_t gbase = ex & ((1ull << D_MISS_SHIFT) - 1);
    const uint32_t mbase = (uint32_t)(ex >> D_MISS_SHIFT);
    const bool overflow = gbase + tile_bytes > (uint64_t)P.out_cap;

    // ---- per-query outputs ---------------------------------------------------------------------
    if (qi < nq) {
        r_out_off[q0 + qi] = (uint32_t)(gbase + my_o);
        r_out_len[q0 + qi] = (uint16_t)my_len;
        r_status[q0 + qi] = r.status;
        if (my_miss) r_miss_idx[mbase + my_mrank] = q0 + qi;
        if (MULTI && r_qidx_out) r_qidx_out[q0 + qi] = qidx;
    }
    if (overflow && tid == 0) r_totals[2] = P.epoch;

    // ---- emit ---------------------------------------------------------------------------------------
    // Responses are assembled in (swizzled) shared memory and flushed with aligned 16-byte stores: scattered 4-byte stores
    // straight to global memory cost one L1->L2 request per lane, and that request path — not DRAM, not the ALUs — is what
    // a tile of ~300-byte service answers saturates.  A tile whose responses fit one staging window (128 x 64-byte answers
    // do) is one round: every thread writes its response, all flush.
    // A BIG tile in the service variant of the kernel (SVC) goes through the window in ROUNDS and splits the work so that all
    // 128 threads stay busy with independent loads.  Round k = the responses that START in bytes [k*WIN, (k+1)*WIN) of the
    // tile (each at most MAXRESP long, which the buffer allows for past the window).  Their threads write the header and the
    // question; the rest of a service answer — the children's ready RRs — became copy jobs of at most 64 bytes
    // (plan_service) that ANY thread runs, a thread per job: a thread walking its own service record child by child is one
    // dependent DRAM round trip after another, and warps of mixed answer sizes idle most lanes.  The jobs of thread t sit
    // at the exclusive prefix of the job counts (the second field of the CTA scan), so the list is sorted by tile offset and
    // a round's jobs are one contiguous run of it — a round touches only its own jobs.
    // Without SVC a big tile writes straight to global memory, thread per response; so does, in either variant, a tile with a
    // query on the generic byte path or a response over MAXRESP (TCP).
    const bool odd_emit = my_len && (!(r.sp && !r.trunc) || my_len > (uint32_t)MAXRESP);
    const bool direct = __syncthreads_or(odd_emit) || (!SVC && tile_bytes > (uint32_t)WIN);
    if (!overflow && direct) {
        // `out` may be pinned host memory (zero-copy results): 4-byte stores over PCIe would be ruinous,
        // so such tiles assemble in the device bounce buffer and then move their contiguous range with
        // coalesced 16-byte stores (the bytes are still in L2)
        uint8_t* const dst = r_bounce ? r_bounce : r_out;
        if (my_len) {
            if (!(r.sp && !r.trunc)) emit_response(P, r, dst + gbase + my_o, qidx);
            else { WrT<2> w; w.begin_global(dst, (uint32_t)(gbase + my_o)); emit_fast(P, r, w, qidx); }
        }
        STAMP(9);
        if (r_bounce && tile_bytes) {
            __syncthreads();
            const uint8_t* src = r_bounce + gbase;
            uint8_t* g = r_out + gbase;
            uint32_t head = (uint32_t)((16 - (gbase & 15)) & 15);
            if (head > tile_bytes) head = tile_bytes;
            if (tid < (int)head) g[tid] = src[tid];
            const uint32_t nv = (tile_bytes - head) >> 4;
            for (uint32_t i = tid; i < nv; i += T) *(uint4*)(g + head + 16 * i) = *(const uint4*)(src + head + 16 * i);
            const uint32_t x0 = head + (nv << 4);
            if (x0 + tid < tile_bytes) g[x0 + tid] = src[x0 + tid];
        }
    } else if (!overflow && SVC && tile_bytes > (uint32_t)WIN) {
        const uint32_t s_out_a = (uint32_t)__cvta_generic_to_shared(s_out);
        const uint32_t nr = (tile_bytes + WIN - 1) / WIN;                     // <= NROUNDS
        const uint32_t kr = my_o / WIN;
        bool jobs = false;
        if (tid < 4) s_opt[tid] = tid == 0 ? 0x04290000u : tid == 1 ? 0x000000B0u : 0u;          // OPT: 00 | 00 29 | 04 B0 | ttl 0 | rdlen 0, zero padded
        if (tid <= NROUNDS) { s_rstart[tid] = 0xFFFFFFFFu; s_tstart[tid] = 0xFFFFFFFFu; }
        if (tid == 0) s_tstart[NROUNDS + 1] = min(ttot, (uint32_t)TASKCAP);
        __syncthreads();
        if (my_len) { atomicMin(&s_rstart[kr], my_o); atomicMin(&s_tstart[kr], tbase); }         // where each round's responses and jobs start
        if (my_cnt) {
            // the list holds the jobs of the threads in front of the first one whose jobs do not fit; that thread and
            // the ones behind it (their prefixes are larger still) write their responses themselves
            if (tbase + my_cnt <= (uint32_t)TASKCAP) {
                TaskFill fill = { s_task + tbase };
                plan_service(P, r, qidx, my_o, (uint32_t)__cvta_generic_to_shared(s_opt), fill);
                jobs = true;
            } else atomicMin(&s_tstart[NROUNDS + 1], tbase);
        }
        __syncthreads();
        const uint32_t tv = s_tstart[NROUNDS + 1];
        uint8_t* const g = r_out + gbase;
#pragma unroll 1
        for (uint32_t k = 0; k < nr; k++) {
            uint32_t x0 = s_rstart[k], x1 = tile_bytes;                       // this round's byte range of the tile
            if (x0 == 0xFFFFFFFFu) continue;                                  // no response starts in this window (uniform)
            uint32_t t0 = min(s_tstart[k], tv), t1 = tv;                      // and its run of the job list
            for (uint32_t j = k + 1; j < nr; j++) if (s_rstart[j] != 0xFFFFFFFFu) { x1 = s_rstart[j]; t1 = min(s_tstart[j], tv); break; }
            const uint32_t shift = (uint32_t)((gbase + x0) & 15);             // same 16-byte phase in shared and global memory
            const uint32_t delta = shift - x0;                                // tile byte x <-> s_out[delta + x]: a linear buffer
            uint32_t head = (16u - shift) & 15u;                              // up to 16-byte alignment of the global address
            if (head > x1 - x0) head = x1 - x0;
            const uint32_t nz = (shift + (x1 - x0) + 15) >> 4;                // pieces are OR-ed into a zeroed buffer
            for (uint32_t i = tid; i < nz; i += T) ((uint4*)s_out)[i] = make_uint4(0, 0, 0, 0);
            __syncthreads();
            if (my_len && kr == k) {
                WrT<4> w; w.begin(s_out_a, delta + my_o);
                if (jobs) { emit_head_w(r, w); w.end(); } else emit_fast(P, r, w, qidx);
            }
            run_tasks(P, s_task, t0, t1, (uint32_t)tid, s_out_a + delta);
            // The round's bytes leave as ONE bulk copy shared -> global (16-byte aligned on both sides: the buffer keeps the
            // global address's phase), issued by one thread; the partial chunks at both ends go out as bytes.  Results
            // in pinned host memory (zero-copy, P.bounce set) keep the 16-byte stores of all threads.
#ifdef BB_NO_BULK_FLUSH        /* experiment switch: every thread's 16-byte stores instead of the bulk copy */
            const bool bulk = false;
#else
            const bool bulk = r_bounce == nullptr;
#endif
            if (bulk) fence_async_smem();                                     // this thread's writes, for the copy engine
            __syncthreads();
            if (tid < (int)head) g[x0 + tid] = s_out[delta + x0 + tid];
            x0 += head;
            const uint32_t nv = (x1 - x0) >> 4;
            if (bulk) { if (tid == 0 && nv) { bulk_s2g(g + x0, s_out_a + delta + x0, nv << 4); bulk_wait_read(); } }
            else for (uint32_t i = tid; i < nv; i += T) *(uint4*)(g + x0 + 16 * i) = *(const uint4*)(s_out + delta + x0 + 16 * i);
            x0 += nv << 4;
            if (x0 + tid < x1) g[x0 + tid] = s_out[delta + x0 + tid];
            if (k + 1 < nr) __syncthreads();                                  // the buffer is reused by the next round (thread 0 arrives once the engine has read it)
        }
        STAMP(9);
    } else if (!overflow && tile_bytes) {
        const uint32_t shift = (uint32_t)(gbase & 15);                       // same 16-byte phase in shared and global memory
        if (my_len) { WrT<1> w; w.begin((uint32_t)__cvta_generic_to_shared(s_out), shift + my_o); emit_fast(P, r, w, qidx); }
        __syncthreads();
        STAMP(9);
        uint8_t* g = r_out + gbase;                                           // g[x] <-> s_out[swz(shift + x)]
        uint32_t x0 = 0;
        const uint32_t x1 = tile_bytes;
        uint32_t head = (uint32_t)((16 - (gbase & 15)) & 15);                 // up to 16-byte alignment of the global address
        if (head > x1) head = x1;
        if (tid < (int)head) g[tid] = s_out[swz(shift + tid)];
        x0 = head;
        const uint32_t nv = (x1 - x0) >> 4;
        for (uint32_t i = tid; i < nv; i += T) *(uint4*)(g + x0 + 16 * i) = *(const uint4*)(s_out + swz(shift + x0 + 16 * i));
        x0 += nv << 4;
        if (x0 + tid < x1) g[x0 + tid] = s_out[swz(shift + x0 + tid)];
    }

    STAMP(10);
    }   // tile < ntiles
    // ---- self-cleaning: the last block to finish publishes the totals and resets the placement
    // state for the next launch (blocks beyond ntiles only take part in this count) ------------
    if (warp == 0) {
        uint32_t last = 0;
        // ORDERED: this tile's descriptor store must be visible before it counts itself done.  Arrival
        // packing needs no fence here: the claim was an atomic whose return value this thread already
        // consumed, so it has been performed at L2.
        if (lane == 0) { if (ORDERED) __threadfence(); last = atomicAdd(r_counter + 1, 1u) == gridDim.x - 1; }
        last = __shfl_sync(0xffffffffu, last, 0);
        if (last) {                                // every tile has finished reading descriptors / claiming
            __threadfence();
            volatile unsigned long long* D = r_desc;
            unsigned long long cur = 0;
            if (ORDERED) { if (ntiles) cur = D[ntiles - 1] & D_VAL; }            // inclusive prefix of the last tile
            else cur = D[P.ntiles_cap];
            if (lane == 0) {
                const uint32_t tb = (uint32_t)(cur & ((1ull << D_MISS_SHIFT) - 1));
                r_out_off[n] = tb; r_totals[0] = tb; r_totals[1] = (uint32_t)(cur >> D_MISS_SHIFT); r_totals[3] = P.epoch;
                // one 16-byte store (one PCIe write, no fence, nothing waits for it): what the host picks the next batch's variant from
                if (!MULTI && P.fb) *(uint4*)P.fb = make_uint4(tb, n, 0u, P.epoch);
                if (MULTI) {                   // what a host reading only the totals needs to know about the region
                    r_totals[4] = n; r_totals[5] = r_n_dev ? r_n_dev[3] : 0u; r_totals[6] = P.err_in ? *(volatile const uint32_t*)P.err_in : 0u;
                }
            }
            __syncwarp();
            if (ORDERED) { for (uint32_t i = lane; i < ntiles; i += 32) r_desc[i] = 0; }
            else if (lane == 0) r_desc[P.ntiles_cap] = 0;
            if (lane == 0) r_counter[1] = 0;
        }
    }
}


// ---- multi-GPU: route + push ----------------------------------------------------------------
// Ingress side of the sharded design (SURVEY.md §8e).  Each query is parsed just far enough to
// know its lookup key (the same code as resolve, in route mode) and is then written straight
// into the receive region (this rank -> owner rank) in the OWNER's HBM with peer-to-peer stores
// over NVLink: no staging buffer, no separate collective.  Space inside a region is claimed
// with sender-local atomics (a region has exactly one writer rank), so nothing atomic ever
// crosses the link.  A region is laid out as an ordinary batch (packed packets + u32 offsets)
// plus the original query index of each packet, so the owner resolves it with resolve_kernel.
constexpr int MAX_RANKS = 8;
constexpr int PUSH_CNT_SHIFT = 40;
struct PushParams {
    Params P;                              // pkts, pkt_off, n, eng, route = 1, nranks, rank
    uint8_t* region[MAX_RANKS];            // region (rank -> d) inside rank d's receive buffer (peer-mapped)
    uint32_t cap_q, cap_b;                 // capacity of one region: queries, packet bytes
    unsigned long long* cursor;            // [nranks], local: count << 40 | bytes
    uint32_t* done;                        // finished-block counter
    uint32_t* err;                         // set when a region overflows
    uint32_t qidx_base, epoch;
};
__host__ __device__ inline size_t region_off_array(uint32_t) { return 16; }
__host__ __device__ inline size_t region_qidx_array(uint32_t cap_q) { return 16 + 4 * ((size_t)cap_q + 1); }
__host__ __device__ inline size_t region_bytes(uint32_t cap_q) { return (16 + 4 * ((size_t)cap_q + 1) + 4 * (size_t)cap_q + 15) & ~(size_t)15; }
__host__ __device__ inline size_t region_size(uint32_t cap_q, uint32_t cap_b) { return (region_bytes(cap_q) + cap_b + 64 + 255) & ~(size_t)255; }

__global__ void __launch_bounds__(T, BB_MIN_BLOCKS) route_push_kernel(const PushParams A) {
    const Params& P = A.P;
    // the packets start 16 bytes in: a staged packet's shared address is never 0 (Res::sp == 0 means "not staged")
    __shared__ __align__(16) uint8_t s_inbuf[16 + S_IN + 32];
    uint8_t* const s_in = s_inbuf + 16;
    __shared__ __align__(16) uint8_t s_sorted[S_IN + 16 * MAX_RANKS + 32];     // the tile's packets grouped by owner
    __shared__ uint32_t s_moff[T], s_mq[T];                                    // per-owner-grouped offsets / query indices
    __shared__ uint32_t s_off[T + 1];
    // per (tile, owner): queries << 24 | packet bytes.  One 32-bit word so that the claim is a native shared-memory
    // add (a 64-bit one is a compare-and-swap loop, and the whole tile contends on nranks words).
    // <= 128 queries of <= 65535 bytes each: the byte field stays below 2^24.
    __shared__ uint32_t s_cur[MAX_RANKS];
    __shared__ unsigned long long s_base[MAX_RANKS];
    __shared__ uint32_t s_kstart[MAX_RANKS + 1], s_bstart[MAX_RANKS];
    __shared__ uint32_t s_ovf;
    __shared__ __align__(16) uint8_t s_sfx[256];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    for (int i = tid; i < 64; i += T) ((uint32_t*)s_sfx)[i] = __ldg((const uint32_t*)P.eng->wire_tail + i);
    if (tid < MAX_RANKS) s_cur[tid] = 0;
    if (tid == 0) s_ovf = 0;
    STAMP(0);
    const uint32_t q0 = blockIdx.x * T;
    const uint32_t nq = min((uint32_t)T, P.n - q0);
    for (int i = tid; i <= (int)nq; i += T) s_off[i] = P.pkt_off[q0 + i];
    __syncthreads();
    STAMP(1);
    const uint32_t b0 = s_off[0], b1 = s_off[nq];
    const uint32_t a0 = b0 & ~15u;
    const bool staged = b1 >= b0 && b1 - a0 <= S_IN;
    if (staged) {
        const uint4* src = (const uint4*)(P.pkts + a0);
        uint4* dst = (uint4*)s_in;
        const uint32_t nv = (b1 - a0 + 15) >> 4;
        for (uint32_t i = tid; i < nv; i += T) dst[i] = __ldg(src + i);
    }
    __syncthreads();
    STAMP(2);
    Res r;
    r.owner = (uint8_t)P.rank;                     // queries that need no lookup are answered where they arrived
    r.sp = 0; r.p = nullptr;
    uint32_t len = 0, k = 0, boff = 0;
    const bool have = tid < (int)nq;
    if (have) {
        const uint32_t o0 = s_off[tid], o1 = s_off[tid + 1];
        if (o0 >= b0 && o1 >= o0 && o1 <= b1 && o1 - o0 <= 65535u) {
            len = o1 - o0;
            r.p = staged ? s_in + (o0 - a0) : P.pkts + o0;
            r.sp = staged ? (uint32_t)__cvta_generic_to_shared(s_in) + (o0 - a0) : 0u;
            resolve_query(P, r, len, 0, (uint32_t)__cvta_generic_to_shared(s_sfx));
            if (r.owner >= P.nranks) r.owner = (uint8_t)P.rank;
        }
        const uint32_t old = atomicAdd(&s_cur[r.owner], (1u << 24) | len);
        k = old >> 24; boff = old & 0xFFFFFFu;
    }
    __syncthreads();
    STAMP(6);
    // one claim per (tile, owner) in the sender-local cursor of region (this rank -> owner)
    if (tid < (int)P.nranks) {
        const uint32_t t = s_cur[tid];
        s_base[tid] = t ? atomicAdd(A.cursor + tid, ((unsigned long long)(t >> 24) << PUSH_CNT_SHIFT) | (t & 0xFFFFFFu)) : 0ull;
    }
    __syncthreads();
    if (tid == 0) {
        uint32_t kk = 0, bb = 0;
        for (uint32_t d = 0; d < P.nranks; d++) {
            const uint32_t t = s_cur[d]; const unsigned long long base = s_base[d];
            const uint32_t cnt = t >> 24, nb = t & 0xFFFFFFu;
            const uint32_t gk = (uint32_t)(base >> PUSH_CNT_SHIFT);
            const unsigned long long gb = base & ((1ull << PUSH_CNT_SHIFT) - 1);
            if (cnt && (gk + cnt > A.cap_q || gb + nb > A.cap_b)) { s_ovf = 1; *A.err = 1; }
            s_kstart[d] = kk; kk += cnt;
            bb += (uint32_t)((gb - bb) & 15);      // group start has the 16-byte phase of its destination
            s_bstart[d] = bb; bb += nb;
        }
        s_kstart[P.nranks] = kk;
    }
    __syncthreads();
    const bool ovf = s_ovf != 0;
    STAMP(7);
    if (have && !ovf) {
        const unsigned long long base = s_base[r.owner];
        const uint32_t gb = (uint32_t)(base & ((1ull << PUSH_CNT_SHIFT) - 1)) + boff;
        if (staged) {
            s_moff[s_kstart[r.owner] + k] = gb;
            s_mq[s_kstart[r.owner] + k] = A.qidx_base + q0 + tid;
            WrT<0, true> w; w.begin((uint32_t)__cvta_generic_to_shared(s_sorted), s_bstart[r.owner] + boff);
            w.copy(r.sp, len);
            w.end();
        } else {                                   // oversized tile: plain peer stores from global memory
            const uint32_t gk = (uint32_t)(base >> PUSH_CNT_SHIFT) + k;
            uint8_t* reg = A.region[r.owner];
            ((uint32_t*)(reg + region_off_array(A.cap_q)))[gk] = gb;
            ((uint32_t*)(reg + region_qidx_array(A.cap_q)))[gk] = A.qidx_base + q0 + tid;
            uint8_t* dst = reg + region_bytes(A.cap_q) + gb;
            const uint8_t* src = P.pkts + s_off[tid];
            for (uint32_t i = 0; i < len; i++) dst[i] = src[i];
        }
    }
    __syncthreads();
    STAMP(8);
    if (staged && !ovf) {
        // per owner: one contiguous chunk of packets and of metadata, pushed with coalesced peer stores
        for (uint32_t d = 0; d < P.nranks; d++) {
            const uint32_t t = s_cur[d]; const unsigned long long base = s_base[d];
            const uint32_t cnt = t >> 24, nb = t & 0xFFFFFFu;
            if (!cnt) continue;
            uint8_t* reg = A.region[d];
            const uint32_t gk = (uint32_t)(base >> PUSH_CNT_SHIFT);
            const unsigned long long gb = base & ((1ull << PUSH_CNT_SHIFT) - 1);
            uint32_t* go = (uint32_t*)(reg + region_off_array(A.cap_q)) + gk;
            uint32_t* gq = (uint32_t*)(reg + region_qidx_array(A.cap_q)) + gk;
            for (uint32_t i = tid; i < cnt; i += T) { go[i] = s_moff[s_kstart[d] + i]; gq[i] = s_mq[s_kstart[d] + i]; }
            uint8_t* g = reg + region_bytes(A.cap_q) + gb;                    // g[x] <-> s_sorted[s_bstart[d] + x]
            const uint8_t* sm = s_sorted + s_bstart[d];
            uint32_t x0 = 0;
            uint32_t head = (uint32_t)((16 - (gb & 15)) & 15);
            if (head > nb) head = nb;
            if (tid < (int)head) g[tid] = sm[tid];
            x0 = head;
            const uint32_t nv = (nb - x0) >> 4;
            for (uint32_t i = tid; i < nv; i += T) *(uint4*)(g + x0 + 16 * i) = *(const uint4*)(sm + x0 + 16 * i);
            x0 += nv << 4;
            if (x0 + tid < nb) g[x0 + tid] = sm[x0 + tid];
        }
    }
    // The last block publishes the region headers (count, bytes, end-of-offsets sentinel) and then,
    // with a system-scope release store, the epoch flag the owner's wait kernel acquires: the exchange
    // needs no collective, only this ordered pair of peer stores per (source, owner).
    // A block orders its peer stores before its done count with a device-scope fence only (the barrier
    // orders every thread's stores before thread 0's fence; fences are cumulative).  The system-scope
    // release is the last block's alone: it has observed every other block's count, so by causality
    // order all their stores precede its flag store for whoever acquires the flag at system scope.
    __syncthreads();
    STAMP(9);
    if (warp == 0) {
        uint32_t last = 0;
        if (lane == 0) { __threadfence(); last = atomicAdd(A.done, 1u) == gridDim.x - 1; }
        STAMP(10);
        last = __shfl_sync(0xffffffffu, last, 0);
        if (last && lane < (int)P.nranks) {
            __threadfence();
            const unsigned long long c = *(volatile unsigned long long*)(A.cursor + lane);
            const uint32_t cnt = min((uint32_t)(c >> PUSH_CNT_SHIFT), A.cap_q);
            const uint32_t nb = (uint32_t)min(c & ((1ull << PUSH_CNT_SHIFT) - 1), (unsigned long long)A.cap_b);
            uint8_t* reg = A.region[lane];
            ((uint32_t*)(reg + region_off_array(A.cap_q)))[cnt] = nb;
            volatile uint32_t* hdr = (volatile uint32_t*)reg;
            hdr[0] = cnt; hdr[1] = nb; hdr[3] = *A.err;
            // the flag, released at system scope: everything above (and, by cumulativity, every other block's peer stores
            // this thread has observed through the done counter) is visible to whoever acquires it
            asm volatile("st.release.sys.global.u32 [%0], %1;" :: "l"(reg + 8), "r"(A.epoch) : "memory");
            if (P.stage_log && lane == 0) P.stage_log[(size_t)gridDim.x * NSTAGE] = gtime();   // one extra row: flag published
            A.cursor[lane] = 0;
        }
        if (last && lane == 0) *A.done = 0;
    }
}

// Owner side: wait (bounded) until every source rank has published `epoch` in its region header.
__global__ void wait_regions_kernel(const uint8_t* recv_set, size_t reg_size, uint32_t nranks, uint32_t epoch, uint32_t* err) {
    const uint32_t r = threadIdx.x;
    if (r < nranks) {
        const uint32_t* flag = (const uint32_t*)(recv_set + (size_t)r * reg_size) + 2;
        unsigned long long spins = 0;
        for (;;) {                                                // acquire at system scope: pairs with the sender's st.release.sys
            uint32_t v;
            asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(flag) : "memory");
            if (v == epoch) break;
            if (++spins > (1ull << 28)) { *err = 2; break; }      // ~seconds: a peer died; fail instead of hanging
            __nanosleep(64);
        }
    }
}

// Incremental zone update: overwrite the listed 32-byte slots (one thread per 16-byte chunk).  Runs with no
// batch in flight (bb_engine_apply_update synchronises first), so a reader never sees half a slot.
__global__ void patch_slots_kernel(Slot* table, const uint32_t* idx, const uint4* data, uint32_t n) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t < 2u * n) ((uint4*)(table + idx[t >> 1]))[t & 1u] = data[t];
}

}  // namespace bbk

// =================================================================================================
// host side of the C ABI
// =================================================================================================
static thread_local std::string g_cuda_err;
#define CK(call) do { cudaError_t _e = (call); if (_e != cudaSuccess) { g_cuda_err = std::string(#call) + ": " + cudaGetErrorString(_e); return BB_ERR_CUDA; } } while (0)

namespace {
constexpr int NSLOTS = 4;
struct SlotCtx {
    cudaStream_t stream = nullptr; cudaEvent_t ev = nullptr;
    uint8_t* d_pkts = nullptr; uint32_t* d_off = nullptr; uint8_t* d_out = nullptr; uint32_t* d_out_off = nullptr;
    uint8_t* d_status = nullptr; uint32_t* d_miss = nullptr; uint32_t* d_totals = nullptr; uint16_t* d_out_len = nullptr;
    unsigned long long* d_desc = nullptr;        // [ntiles_max] + counter
    uint32_t* h_totals = nullptr;                // pinned
    // pending call
    bool busy = false, zero_copy = false; uint32_t n = 0, epoch = 0;
    const void* zc_seen[5] = {}; bool zc_ok = false;        // last output pointer set checked for being pinned
    uint8_t* out = nullptr; uint32_t out_cap = 0; uint32_t* miss_idx = nullptr; uint32_t* n_miss = nullptr;
};
}

struct bb_engine {
    bb::EngineConst hconst; bb::EngineConst* d_const = nullptr;
    bb::Slot* d_table = nullptr; uint8_t* d_arena = nullptr; uint32_t mask = 0; int ready = 0;
    int device = 0, ordered = 0; uint32_t max_batch = 0, max_bytes = 0, out_dev_cap = 0, max_tiles = 0;
    SlotCtx slots[NSLOTS];
    // look-back / claim scratch of bb_resolve_batch_device, one per caller stream (launches on
    // different streams may overlap)
    static constexpr int MAX_DEV_STREAMS = 16;
    void* dev_stream[MAX_DEV_STREAMS] = {}; unsigned long long* dev_desc[MAX_DEV_STREAMS] = {}; int n_dev_streams = 0;
    uint64_t launches = 0, epoch = 0;
    unsigned long long* stage_log = nullptr;
    // kernel variant per batch (bb_engine_set_kernel_profile): 0 = by the mean response size of the latest finished batch
    int profile = 0; uint32_t mean_resp = 0;
    static constexpr int FB = 64;                                // feedback ring (pinned): {response bytes, queries, -, epoch} written by a launch's last block
    uint32_t* h_fb = nullptr;
    // the zone this engine last synchronised with (incremental updates only continue from that state)
    const bb_zone* zone = nullptr; uint64_t zone_gen = 0; uint64_t arena_cap = 0;
};

extern "C" {

const char* bb_strerror(int err) {
    switch (err) {
    case BB_OK: return "ok";
    case BB_ERR_ARG: return "invalid argument";
    case BB_ERR_SNAPSHOT: return "snapshot is not valid JSON-lines (or repeats a path)";
    case BB_ERR_CUDA: return "CUDA error";
    case BB_ERR_NOMEM: return "out of memory";
    case BB_ERR_CAPACITY: return "output capacity too small for this batch";
    case BB_ERR_NO_DEVICE: return "no CUDA device (binder_b200 has no CPU fallback)";
    case BB_ERR_DOMAIN: return "dns_domain must be a lower-case, encodable DNS name";
    case BB_ERR_PROTOCOL: return "balancer frame stream: unknown frame type, INBOUND_TCP, or oversized packet";
    }
    return "unknown error";
}
const char* bb_last_cuda_error(void) { return g_cuda_err.c_str(); }
int bb_abi_version(void) { return BB_ABI_VERSION; }

void* bb_host_alloc(size_t bytes) { void* p = nullptr; return cudaMallocHost(&p, bytes ? bytes : 1) == cudaSuccess ? p : nullptr; }
void bb_host_free(void* p) { if (p) cudaFreeHost(p); }

static int engine_alloc(bb_engine* e) {
    CK(cudaSetDevice(e->device));
    CK(cudaMalloc(&e->d_const, sizeof(bb::EngineConst)));
    CK(cudaMemcpy(e->d_const, &e->hconst, sizeof(bb::EngineConst), cudaMemcpyHostToDevice));
    e->max_tiles = (e->max_batch + bbk::T - 1) / bbk::T;
    CK(cudaMallocHost(&e->h_fb, bb_engine::FB * 16));
    memset(e->h_fb, 0, bb_engine::FB * 16);
    if (const char* pf = getenv("BB_PROFILE")) e->profile = !strcmp(pf, "small") ? 1 : !strcmp(pf, "service") ? 2 : 0;
    uint64_t cap = (uint64_t)e->max_batch * 512;                 // device-side response buffer per slot
    if (cap < (1u << 20)) cap = 1u << 20;
    if (cap > 0xFFFFFF00ull) cap = 0xFFFFFF00ull;
    e->out_dev_cap = (uint32_t)cap;
    for (auto& s : e->slots) {
        CK(cudaStreamCreateWithFlags(&s.stream, cudaStreamNonBlocking));
        CK(cudaEventCreateWithFlags(&s.ev, cudaEventDisableTiming));
        CK(cudaMalloc(&s.d_pkts, (size_t)e->max_bytes + 64));
        CK(cudaMalloc(&s.d_off, ((size_t)e->max_batch + 1) * 4));
        CK(cudaMalloc(&s.d_out, (size_t)e->out_dev_cap + 64));
        CK(cudaMalloc(&s.d_out_off, ((size_t)e->max_batch + 1) * 4));
        CK(cudaMalloc(&s.d_status, (size_t)e->max_batch + 16));
        CK(cudaMalloc(&s.d_out_len, (size_t)e->max_batch * 2 + 16));
        CK(cudaMalloc(&s.d_miss, (size_t)e->max_batch * 4 + 16));
        CK(cudaMalloc(&s.d_totals, 16));
        CK(cudaMalloc(&s.d_desc, ((size_t)e->max_tiles + 4) * 8));
        CK(cudaMemset(s.d_desc, 0, ((size_t)e->max_tiles + 4) * 8));
        CK(cudaMemset(s.d_totals, 0, 16));
        CK(cudaMallocHost(&s.h_totals, 16));
    }
    return BB_OK;
}

bb_engine* bb_engine_create(const bb_engine_opts* o, int* err) {
    auto fail = [&](int c) -> bb_engine* { if (err) *err = c; return nullptr; };
    if (err) *err = BB_OK;
    if (!o || !o->dns_domain) return fail(BB_ERR_ARG);
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0) return fail(BB_ERR_NO_DEVICE);
    if (o->device < 0 || o->device >= ndev) return fail(BB_ERR_ARG);
    bb_engine* e = new bb_engine();
    if (!bb::make_engine_const(o->dns_domain, o->recursion != 0, e->hconst)) { delete e; return fail(BB_ERR_DOMAIN); }
    // A probe wants ONE 32-byte sector of a table far larger than L2; by default an L2 miss fetches 128 bytes from
    // DRAM around it (measured: tools/micro/probe_gran.cu, 4 sectors of dram__bytes_read per sector asked for).
    // Sector-granular fetches cut the probe's DRAM traffic 4x; streaming reads ask for whole lines anyway.
    if (cudaSetDevice(o->device) == cudaSuccess) {
        const char* gr = getenv("BB_L2_GRAN");                     // experiments: 32 (default), 64, 128
        cudaDeviceSetLimit(cudaLimitMaxL2FetchGranularity, gr ? (size_t)atoi(gr) : 32);
    }
    cudaGetLastError();
    e->device = o->device; e->ordered = o->ordered_output ? 1 : 0;
    e->max_batch = o->max_batch ? o->max_batch : (1u << 20);
    if (e->max_batch > (1u << 22)) { delete e; return fail(BB_ERR_ARG); }
    e->max_bytes = o->max_batch_bytes ? o->max_batch_bytes : e->max_batch * 64;
    int rc = engine_alloc(e);
    if (rc != BB_OK) { bb_engine_destroy(e); return fail(rc); }
    return e;
}

void bb_engine_destroy(bb_engine* e) {
    if (!e) return;
    cudaSetDevice(e->device);
    cudaDeviceSynchronize();
    for (auto& s : e->slots) {
        cudaFree(s.d_pkts); cudaFree(s.d_off); cudaFree(s.d_out); cudaFree(s.d_out_off); cudaFree(s.d_status); cudaFree(s.d_out_len);
        cudaFree(s.d_miss); cudaFree(s.d_totals); cudaFree(s.d_desc); if (s.h_totals) cudaFreeHost(s.h_totals);
        if (s.ev) cudaEventDestroy(s.ev); if (s.stream) cudaStreamDestroy(s.stream);
    }
    for (int i = 0; i < e->n_dev_streams; i++) cudaFree(e->dev_desc[i]);
    cudaFree(e->d_const); cudaFree(e->d_table); cudaFree(e->d_arena);
    if (e->h_fb) cudaFreeHost(e->h_fb);
    delete e;
}

int bb_engine_swap_zone(bb_engine* e, const bb_zone* z) {
    if (!e || !z) return BB_ERR_ARG;
    const bb::ZoneImage* img = bb_zone_image(z);
    CK(cudaSetDevice(e->device));
    bb::Slot* nt = nullptr; uint8_t* na = nullptr;
    // head room in the arena: updates append re-derived records (bb_engine_apply_update)
    const uint64_t cap = img->arena_len + (img->arena_len / 2 > (4u << 20) ? img->arena_len / 2 : (4u << 20));
    CK(cudaMalloc(&nt, (size_t)img->nslots * sizeof(bb::Slot)));
    CK(cudaMalloc(&na, (size_t)cap + 64));
    CK(cudaMemcpy(nt, img->slots, (size_t)img->nslots * sizeof(bb::Slot), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(na, img->arena, (size_t)img->arena_len, cudaMemcpyHostToDevice));
    CK(cudaDeviceSynchronize());                 // batches in flight finish on the old epoch
    bb::Slot* ot = e->d_table; uint8_t* oa = e->d_arena;
    e->d_table = nt; e->d_arena = na; e->mask = img->nslots - 1; e->ready = img->ready; e->arena_cap = cap;
    cudaFree(ot); cudaFree(oa);
    // the zone's pending-change list restarts here (a zone feeds one engine incrementally)
    bb_zone_mark_synced(const_cast<bb_zone*>(z));
    e->zone = z; e->zone_gen = bb_zone_sync_gen(z);
    return BB_OK;
}

// After bb_zone_apply: ship what changed — the touched 32-byte slots and the arena tail — instead of the
// whole image.  Falls back to a full swap when the table was laid out again, the arena outgrew its
// device allocation, or this engine is not the one that took the zone's previous changes.
int bb_engine_apply_update(bb_engine* e, bb_zone* z) {
    if (!e || !z) return BB_ERR_ARG;
    const bb::ZoneImage* img = bb_zone_image(z);
    const uint32_t* slots = nullptr; uint32_t n = 0; uint64_t from = 0; int relaid = 0;
    if (bb_zone_pending(z, &slots, &n, &from, &relaid) != BB_OK) return BB_ERR_ARG;
    if (relaid || !e->d_table || e->zone != z || e->zone_gen != bb_zone_sync_gen(z) || e->mask != img->nslots - 1 ||
        img->arena_len > e->arena_cap)
        return bb_engine_swap_zone(e, z);
    CK(cudaSetDevice(e->device));
    CK(cudaDeviceSynchronize());                 // batches in flight finish on the old state
    if (img->arena_len > from)
        CK(cudaMemcpy(e->d_arena + from, img->arena + from, (size_t)(img->arena_len - from), cudaMemcpyHostToDevice));
    if (n) {
        std::vector<bb::Slot> data(n);
        for (uint32_t i = 0; i < n; i++) data[i] = img->slots[slots[i]];
        uint32_t* d_idx = nullptr; uint4* d_data = nullptr;
        CK(cudaMalloc(&d_idx, (size_t)n * 4)); 
        if (cudaMalloc(&d_data, (size_t)n * sizeof(bb::Slot)) != cudaSuccess) { cudaFree(d_idx); g_cuda_err = "cudaMalloc (slot patch)"; return BB_ERR_CUDA; }
        cudaError_t c1 = cudaMemcpy(d_idx, slots, (size_t)n * 4, cudaMemcpyHostToDevice);
        cudaError_t c2 = cudaMemcpy(d_data, data.data(), (size_t)n * sizeof(bb::Slot), cudaMemcpyHostToDevice);
        if (c1 == cudaSuccess && c2 == cudaSuccess) {
            bbk::patch_slots_kernel<<<(2 * n + 255) / 256, 256>>>(e->d_table, d_idx, d_data, n);
            c1 = cudaGetLastError(); c2 = cudaDeviceSynchronize();
        }
        cudaFree(d_idx); cudaFree(d_data);
        if (c1 != cudaSuccess || c2 != cudaSuccess) { g_cuda_err = cudaGetErrorString(c1 != cudaSuccess ? c1 : c2); return BB_ERR_CUDA; }
        e->launches++;
    }
    e->ready = img->ready;
    bb_zone_mark_synced(z);
    e->zone_gen = bb_zone_sync_gen(z);
    return BB_OK;
}
// Recursion pre-filter (lib/recursion.js:329-344, SURVEY.md section 8f row 3).  region_domain =
// Recursion's opts.dnsDomain; dc_names = the keys of self.dcs that still have an upstream after the
// "not one of my own addresses" filter (:360-379); ptr_forwardable = any such upstream exists at all.
// With a filter set, a miss Recursion.resolve() would answer REFUSED without asking anyone is answered
// REFUSED by the kernel and never enters miss_idx.  NULL region_domain removes the filter.
int bb_engine_set_recursion_filter(bb_engine* e, const char* region_domain, const char* const* dc_names, uint32_t n_dc,
                                   int ptr_forwardable) {
    if (!e || (n_dc && !dc_names) || n_dc > bb::RF_MAX_DC) return BB_ERR_ARG;
    if (!bb::set_recursion_filter_const(e->hconst, region_domain, dc_names, n_dc, ptr_forwardable != 0)) return BB_ERR_ARG;
    CK(cudaSetDevice(e->device));
    CK(cudaDeviceSynchronize());                                   // batches in flight finish with the old filter
    CK(cudaMemcpy(e->d_const, &e->hconst, sizeof(bb::EngineConst), cudaMemcpyHostToDevice));
    return BB_OK;
}
int bb_engine_is_ready(const bb_engine* e) { return e && e->ready; }
int bb_engine_slots(const bb_engine*) { return NSLOTS; }
int bb_engine_set_kernel_profile(bb_engine* e, int profile) { if (!e || profile < 0 || profile > 2) return BB_ERR_ARG; e->profile = profile; return BB_OK; }
uint32_t bb_engine_max_batch(const bb_engine* e) { return e ? e->max_batch : 0; }
uint32_t bb_engine_max_batch_bytes(const bb_engine* e) { return e ? e->max_bytes : 0; }
uint64_t bb_engine_launch_count(const bb_engine* e) { return e ? e->launches : 0; }
uint32_t bb_engine_launch_epoch(const bb_engine* e) { return e ? (uint32_t)e->epoch : 0; }
void bb_engine_set_stage_log(bb_engine* e, unsigned long long* d_log) { if (e) e->stage_log = d_log; }

static int launch(bb_engine* e, unsigned long long* desc, const uint8_t* d_pkts, const uint32_t* d_off, uint32_t n,
                  uint64_t seed, uint32_t qidx_base, uint8_t* d_out, uint32_t out_cap, uint32_t* d_out_off, uint16_t* d_out_len,
                  uint8_t* d_status, uint32_t* d_miss, uint32_t* d_totals, cudaStream_t st, uint8_t* bounce = nullptr, uint32_t flags = 0,
                  bool feedback = false) {
    bbk::Params P;
    P.pkts = d_pkts; P.pkt_off = d_off; P.n = n; P.seed = seed; P.qidx_base = qidx_base;
    P.out = d_out; P.out_cap = out_cap; P.out_off = d_out_off; P.out_len = d_out_len; P.status = d_status; P.miss_idx = d_miss; P.totals = d_totals;
    P.table = e->d_table; P.mask = e->mask; P.arena = e->d_arena; P.ready = e->ready && e->d_table;
    P.eng = e->d_const; P.suffix_len = e->hconst.suffix_len; P.soa_len = e->hconst.soa_len; P.recursion = e->hconst.recursion; P.lean_ok = e->hconst.lean_ok;
    P.ntiles = (n + bbk::T - 1) / bbk::T;
    P.desc = desc; P.ntiles_cap = e->max_tiles; P.counter = (uint32_t*)(desc + e->max_tiles + 1);
    P.epoch = (uint32_t)(++e->epoch);
    P.stage_log = e->stage_log;
    P.n_dev = nullptr; P.qidx_map = nullptr; P.route = 0; P.nranks = 1; P.rank = 0; P.regions = 0; P.bounce = bounce; P.qidx_out = nullptr; P.err_in = nullptr; P.tcp = (flags & BB_BATCH_TCP) ? 1u : 0u;
    // An empty batch still runs one block: its last-block path writes out_off[0] = 0 and totals {0, 0, -, epoch}, so a
    // caller polling the done marker sees this launch finish like any other (no tiles, so nothing to stamp)
    if (n == 0) P.stage_log = nullptr;
    const uint32_t grid = P.ntiles ? P.ntiles : 1u;
    // Which variant: the service variant (copy jobs + emit rounds, a tile per SM fewer) pays off when answers are long.  Decided
    // from the latest batch whose totals are known: the host path learns them in bb_resolve_wait, the device path from a
    // 16-byte copy of d_totals that follows every launch (looked at only once its epoch has landed: no synchronisation).
    {
        uint32_t best = 0;                                       // the newest launch whose last block has reported
        for (int i = 0; i < bb_engine::FB; i++) {
            const volatile uint32_t* f = e->h_fb + 4 * i;
            const uint32_t ep = f[3];
            if (ep && f[1] && (best == 0 || (int32_t)(ep - best) > 0)) { best = ep; e->mean_resp = f[0] / f[1]; }
        }
    }
    // profile 0: the service variant when the latest known batch averaged >= 96 response bytes per query (its tiles are then
    // "big": more than one staging window, where copy jobs pay off; config 2's 64-byte answers stay on the small variant)
    const bool svc = e->profile == 2 || (e->profile == 0 && e->mean_resp >= 96);
    P.fb = (feedback && e->profile == 0) ? e->h_fb + 4 * (P.epoch % bb_engine::FB) : nullptr;
    // no memsets: the kernel leaves desc/counter zeroed for the next launch (self-cleaning)
    if (svc) {
        if (e->ordered) bbk::resolve_kernel<true, false, true><<<grid, bbk::T, 0, st>>>(P);
        else bbk::resolve_kernel<false, false, true><<<grid, bbk::T, 0, st>>>(P);
    } else {
        if (e->ordered) bbk::resolve_kernel<true, false, false><<<grid, bbk::T, 0, st>>>(P);
        else bbk::resolve_kernel<false, false, false><<<grid, bbk::T, 0, st>>>(P);
    }
    CK(cudaGetLastError());
    e->launches++;
    return BB_OK;
}

int bb_resolve_batch_device(bb_engine* e, const uint8_t* d_pkts, const uint32_t* d_pkt_off, uint32_t n,
                            uint64_t seed, uint32_t qidx_base, uint8_t* d_out, uint32_t out_cap, uint32_t* d_out_off,
                            uint16_t* d_out_len, uint8_t* d_status, uint32_t* d_miss_idx, uint32_t* d_totals, void* stream) {
    if (!e || n > e->max_batch || ((uintptr_t)d_pkts & 15) || ((uintptr_t)d_out & 15)) return BB_ERR_ARG;
    int si = -1;
    for (int i = 0; i < e->n_dev_streams; i++) if (e->dev_stream[i] == stream) si = i;
    if (si < 0) {
        if (e->n_dev_streams == bb_engine::MAX_DEV_STREAMS) return BB_ERR_ARG;
        CK(cudaSetDevice(e->device));
        unsigned long long* dsc = nullptr;
        CK(cudaMalloc(&dsc, ((size_t)e->max_tiles + 4) * 8));
        CK(cudaMemset(dsc, 0, ((size_t)e->max_tiles + 4) * 8));
        si = e->n_dev_streams++; e->dev_stream[si] = stream; e->dev_desc[si] = dsc;
    }
    return launch(e, e->dev_desc[si], d_pkts, d_pkt_off, n, seed, qidx_base, d_out, out_cap, d_out_off, d_out_len, d_status, d_miss_idx,
                  d_totals, (cudaStream_t)stream, nullptr, 0, true);
}

int bb_resolve_submit_ex(bb_engine* e, int slot, const uint8_t* pkts, const uint32_t* pkt_off, uint32_t n, uint64_t seed,
                         uint32_t qidx_base, uint8_t* out, uint32_t out_cap, uint32_t* out_off, uint16_t* out_len, uint8_t* status,
                         uint32_t* miss_idx, uint32_t* n_miss, uint32_t flags) {
    if (!e || slot < 0 || slot >= NSLOTS || !pkt_off || !out_off || !n_miss || (n && (!pkts || !status || !miss_idx || !out_len))) return BB_ERR_ARG;
    SlotCtx& s = e->slots[slot];
    if (s.busy || n > e->max_batch) return BB_ERR_ARG;
    const uint32_t total_in = pkt_off[n];
    if (total_in > e->max_bytes) return BB_ERR_ARG;
    // every tile's byte range must be inside the batch and the ranges in order (the kernel holds each packet to its
    // tile's range): a bad offset array is an argument error, not an illegal address on the device
    for (uint32_t q = 0, prev = 0; q <= n; q += (q + bbk::T <= n || q == n) ? bbk::T : n - q) {
        if (pkt_off[q] < prev || pkt_off[q] > total_in) return BB_ERR_ARG;
        prev = pkt_off[q];
        if (q == n) break;
    }
    CK(cudaSetDevice(e->device));
    if (total_in) CK(cudaMemcpyAsync(s.d_pkts, pkts, total_in, cudaMemcpyHostToDevice, s.stream));
    CK(cudaMemcpyAsync(s.d_off, pkt_off, ((size_t)n + 1) * 4, cudaMemcpyHostToDevice, s.stream));
    // Zero-copy results: when every output buffer is pinned (mapped) host memory — bb_host_alloc — the
    // kernel's coalesced flush writes the responses straight into it over PCIe: no device staging, no
    // D2H copies and no host round trip to learn the sizes.  Otherwise: staged copies (below).
    const void* outs[5] = { out, out_off, out_len, status, miss_idx };
    // (whether the set is pinned does not depend on n: an empty batch must not cache "not pinned" for its buffers)
    if (memcmp(outs, s.zc_seen, sizeof outs) != 0) {
        bool ok = ((uintptr_t)out & 15) == 0;
        for (int i = 0; ok && i < 5; i++) {
            cudaPointerAttributes at;
            ok = cudaPointerGetAttributes(&at, outs[i]) == cudaSuccess && at.type == cudaMemoryTypeHost && at.devicePointer == outs[i];
        }
        cudaGetLastError();
        memcpy(s.zc_seen, outs, sizeof outs); s.zc_ok = ok;
    }
    s.zero_copy = s.zc_ok && n != 0;
    if (s.zero_copy) {
        const uint32_t zcap = out_cap < e->out_dev_cap ? out_cap : e->out_dev_cap;    // the bounce buffer bounds it too
        int rc = launch(e, s.d_desc, s.d_pkts, s.d_off, n, seed, qidx_base, out, zcap, out_off, out_len, status, miss_idx, s.h_totals, s.stream, s.d_out, flags);
        if (rc != BB_OK) return rc;
        CK(cudaEventRecord(s.ev, s.stream));
        s.busy = true; s.n = n; s.epoch = (uint32_t)e->epoch; s.out = out; s.out_cap = out_cap; s.miss_idx = miss_idx; s.n_miss = n_miss;
        return BB_OK;
    }
    uint32_t cap = out_cap < e->out_dev_cap ? out_cap : e->out_dev_cap;
    int rc = launch(e, s.d_desc, s.d_pkts, s.d_off, n, seed, qidx_base, s.d_out, cap, s.d_out_off, s.d_out_len, s.d_status, s.d_miss, s.d_totals, s.stream, nullptr, flags);
    if (rc != BB_OK) return rc;
    CK(cudaMemcpyAsync(s.h_totals, s.d_totals, 16, cudaMemcpyDeviceToHost, s.stream));
    CK(cudaEventRecord(s.ev, s.stream));
    CK(cudaMemcpyAsync(out_off, s.d_out_off, ((size_t)n + 1) * 4, cudaMemcpyDeviceToHost, s.stream));
    if (n) CK(cudaMemcpyAsync(status, s.d_status, n, cudaMemcpyDeviceToHost, s.stream));
    if (n) CK(cudaMemcpyAsync(out_len, s.d_out_len, (size_t)n * 2, cudaMemcpyDeviceToHost, s.stream));
    s.busy = true; s.n = n; s.epoch = (uint32_t)e->epoch; s.out = out; s.out_cap = out_cap; s.miss_idx = miss_idx; s.n_miss = n_miss;
    return BB_OK;
}

int bb_resolve_submit(bb_engine* e, int slot, const uint8_t* pkts, const uint32_t* pkt_off, uint32_t n, uint64_t seed,
                      uint32_t qidx_base, uint8_t* out, uint32_t out_cap, uint32_t* out_off, uint16_t* out_len, uint8_t* status,
                      uint32_t* miss_idx, uint32_t* n_miss) {
    return bb_resolve_submit_ex(e, slot, pkts, pkt_off, n, seed, qidx_base, out, out_cap, out_off, out_len, status, miss_idx, n_miss, 0);
}

int bb_resolve_wait(bb_engine* e, int slot) {
    if (!e || slot < 0 || slot >= NSLOTS) return BB_ERR_ARG;
    SlotCtx& s = e->slots[slot];
    if (!s.busy) return BB_ERR_ARG;
    s.busy = false;
    CK(cudaSetDevice(e->device));
    CK(cudaEventSynchronize(s.ev));
    const uint32_t total = s.n ? s.h_totals[0] : 0, nmiss = s.n ? s.h_totals[1] : 0;
    if (s.n) e->mean_resp = total / s.n;
    const bool ovf = s.n && s.h_totals[2] == s.epoch;
    if (ovf || total > s.out_cap) { cudaStreamSynchronize(s.stream); return BB_ERR_CAPACITY; }
    if (s.zero_copy) { *s.n_miss = nmiss; return BB_OK; }        // everything is already in the caller's buffers
    if (total) CK(cudaMemcpyAsync(s.out, s.d_out, total, cudaMemcpyDeviceToHost, s.stream));
    if (nmiss) CK(cudaMemcpyAsync(s.miss_idx, s.d_miss, (size_t)nmiss * 4, cudaMemcpyDeviceToHost, s.stream));
    CK(cudaStreamSynchronize(s.stream));
    *s.n_miss = nmiss;
    return BB_OK;
}

int bb_resolve_batch_ex(bb_engine* e, const uint8_t* pkts, const uint32_t* pkt_off, uint32_t n, uint64_t seed,
                        uint32_t qidx_base, uint8_t* out, uint32_t out_cap, uint32_t* out_off, uint16_t* out_len, uint8_t* status,
                        uint32_t* miss_idx, uint32_t* n_miss, uint32_t flags) {
    int rc = bb_resolve_submit_ex(e, 0, pkts, pkt_off, n, seed, qidx_base, out, out_cap, out_off, out_len, status, miss_idx, n_miss, flags);
    if (rc != BB_OK) return rc;
    return bb_resolve_wait(e, 0);
}
int bb_resolve_batch(bb_engine* e, const uint8_t* pkts, const uint32_t* pkt_off, uint32_t n, uint64_t seed,
                     uint32_t qidx_base, uint8_t* out, uint32_t out_cap, uint32_t* out_off, uint16_t* out_len, uint8_t* status,
                     uint32_t* miss_idx, uint32_t* n_miss) {
    return bb_resolve_batch_ex(e, pkts, pkt_off, n, seed, qidx_base, out, out_cap, out_off, out_len, status, miss_idx, n_miss, 0);
}

}  // extern "C"

// =================================================================================================
// multi-GPU shard: receive regions in peer-mapped HBM, route + push, region resolves
// =================================================================================================
struct bb_shard {
    bb_engine* e = nullptr; uint32_t nranks = 1, rank = 0, max_batch = 0, cap_q = 0, cap_b = 0;
    size_t reg_size = 0;
    // 2 x nranks regions: set (step & 1), region s = queries pushed by rank s.  Double-buffered so that
    // a fast rank's push of step k+1 never lands in a region a slower owner is still resolving (step k);
    // by the time step k+2 reuses the set, every rank has passed barrier k+1, i.e. finished resolve k.
    uint8_t* recv = nullptr;
    uint8_t* peer_recv[bbk::MAX_RANKS] = {};       // rank d's receive buffer as mapped here
    unsigned long long* cursor = nullptr; uint32_t* done = nullptr; uint32_t* err = nullptr;
    uint32_t epoch = 0;
    // owner side: one output set per source region, each kind contiguous with a fixed stride so that
    // all regions resolve in ONE launch (grid.y = region)
    uint8_t* d_out = nullptr; uint8_t* d_out_off = nullptr; uint8_t* d_out_len = nullptr; uint8_t* d_status = nullptr;
    uint8_t* d_miss = nullptr; uint8_t* d_totals = nullptr; uint8_t* d_desc = nullptr;
    size_t out_stride = 0, off_stride = 0, len_stride = 0, status_stride = 0, miss_stride = 0, totals_stride = 32, desc_stride = 0;
    uint32_t out_cap = 0;
    // optional pinned host mirrors of the result set (same strides): the resolve kernel writes them directly
    uint8_t* h_out = nullptr; uint8_t* h_out_off = nullptr; uint8_t* h_out_len = nullptr; uint8_t* h_status = nullptr;
    uint8_t* h_miss = nullptr; uint8_t* h_totals = nullptr; uint8_t* h_qidx = nullptr;
    bool host = false; uint32_t resolve_epoch = 0;
    // collective exchange (bb_shard_use_exchange_buffers): route+push fills LOCAL send regions (one per destination), the
    // caller moves them with its collective into the receive regions below, resolve reads those
    uint8_t* x_send = nullptr; uint8_t* x_recv = nullptr;
    uint8_t* recv_base() const { return x_recv ? x_recv : recv; }
};

extern "C" {

bb_shard* bb_shard_create(bb_engine* e, uint32_t nranks, uint32_t rank, uint32_t max_batch, uint32_t bytes_per_query, int* err) {
    auto fail = [&](int c) -> bb_shard* { if (err) *err = c; return nullptr; };
    if (err) *err = BB_OK;
    if (!e || nranks == 0 || nranks > bbk::MAX_RANKS || rank >= nranks || max_batch == 0 || max_batch > e->max_batch) return fail(BB_ERR_ARG);
    bb_shard* s = new bb_shard();
    s->e = e; s->nranks = nranks; s->rank = rank; s->max_batch = max_batch;
    // A region must be able to hold a whole ingress batch: queries that need no lookup stay on the
    // ingress rank, and real DNS traffic is skewed (one hot name sends a full batch to one owner).
    s->cap_q = max_batch;
    s->cap_b = s->cap_q * (bytes_per_query ? bytes_per_query : 64);
    s->reg_size = bbk::region_size(s->cap_q, s->cap_b);
    s->out_cap = s->cap_q * 256u;
    auto ck = [&](cudaError_t c) { if (c != cudaSuccess) { g_cuda_err = cudaGetErrorString(c); return false; } return true; };
    auto up = [](size_t v) { return (v + 255) & ~(size_t)255; };
    s->out_stride = up((size_t)s->out_cap + 64); s->off_stride = up(((size_t)s->cap_q + 1) * 4); s->len_stride = up((size_t)s->cap_q * 2 + 16);
    s->status_stride = up((size_t)s->cap_q + 16); s->miss_stride = up((size_t)s->cap_q * 4 + 16); s->desc_stride = up(((size_t)e->max_tiles + 4) * 8);
    bool ok = ck(cudaSetDevice(e->device)) && ck(cudaMalloc(&s->recv, s->reg_size * nranks * 2)) && ck(cudaMemset(s->recv, 0, s->reg_size * nranks * 2)) &&
              ck(cudaMalloc(&s->cursor, 8 * bbk::MAX_RANKS)) && ck(cudaMemset(s->cursor, 0, 8 * bbk::MAX_RANKS)) &&
              ck(cudaMalloc(&s->done, 16)) && ck(cudaMemset(s->done, 0, 16)) &&
              ck(cudaMalloc(&s->d_out, s->out_stride * nranks)) && ck(cudaMalloc(&s->d_out_off, s->off_stride * nranks)) &&
              ck(cudaMalloc(&s->d_out_len, s->len_stride * nranks)) && ck(cudaMalloc(&s->d_status, s->status_stride * nranks)) &&
              ck(cudaMalloc(&s->d_miss, s->miss_stride * nranks)) && ck(cudaMalloc(&s->d_totals, s->totals_stride * nranks)) &&
              ck(cudaMemset(s->d_totals, 0, s->totals_stride * nranks)) &&
              ck(cudaMalloc(&s->d_desc, s->desc_stride * nranks)) && ck(cudaMemset(s->d_desc, 0, s->desc_stride * nranks));
    s->err = s->done ? s->done + 2 : nullptr;
    if (!ok) { bb_shard_destroy(s); return fail(BB_ERR_CUDA); }
    s->peer_recv[rank] = s->recv;
    return s;
}

void bb_shard_destroy(bb_shard* s) {
    if (!s) return;
    cudaSetDevice(s->e->device); cudaDeviceSynchronize();
    for (uint32_t r = 0; r < s->nranks; r++) if (r != s->rank && s->peer_recv[r]) cudaIpcCloseMemHandle(s->peer_recv[r]);
    cudaFree(s->d_out); cudaFree(s->d_out_off); cudaFree(s->d_out_len); cudaFree(s->d_status); cudaFree(s->d_miss);
    cudaFree(s->d_totals); cudaFree(s->d_desc);
    cudaFree(s->recv); cudaFree(s->cursor); cudaFree(s->done);
    cudaFreeHost(s->h_out); cudaFreeHost(s->h_out_off); cudaFreeHost(s->h_out_len); cudaFreeHost(s->h_status);
    cudaFreeHost(s->h_miss); cudaFreeHost(s->h_totals); cudaFreeHost(s->h_qidx);
    delete s;
}

uint32_t bb_shard_ipc_handle_size(void) { return (uint32_t)sizeof(cudaIpcMemHandle_t); }
uint32_t bb_shard_region_capacity(const bb_shard* s) { return s ? s->cap_q : 0; }

int bb_shard_get_ipc_handle(bb_shard* s, void* out) {
    if (!s || !out) return BB_ERR_ARG;
    CK(cudaSetDevice(s->e->device));
    cudaIpcMemHandle_t h;
    CK(cudaIpcGetMemHandle(&h, s->recv));
    memcpy(out, &h, sizeof h);
    return BB_OK;
}

// handles: nranks x bb_shard_ipc_handle_size() bytes, rank-major (this rank's own entry is ignored)
int bb_shard_open_peers(bb_shard* s, const void* handles) {
    if (!s || !handles) return BB_ERR_ARG;
    CK(cudaSetDevice(s->e->device));
    for (uint32_t r = 0; r < s->nranks; r++) {
        if (r == s->rank) continue;
        cudaIpcMemHandle_t h;
        memcpy(&h, (const uint8_t*)handles + (size_t)r * sizeof h, sizeof h);
        void* p = nullptr;
        CK(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
        s->peer_recv[r] = (uint8_t*)p;
    }
    return BB_OK;
}

// Collective exchange instead of peer stores (the NCCL all-to-all baseline of SURVEY.md section 8e): with two caller-owned
// device buffers of bb_shard_exchange_bytes() each, bb_shard_route_push fills LOCAL send regions — region d of the current
// set = what this rank routes to rank d, laid out exactly like a receive region — and bb_shard_resolve (wait_for_peers = 0)
// reads the receive buffer, into which the caller's collective has moved every rank's region for this rank.  The set in use
// alternates per step: set = step parity (bb_shard_exchange_set).  NULL, NULL returns to peer stores.
int bb_shard_use_exchange_buffers(bb_shard* s, void* d_send, void* d_recv) {
    if (!s || (!d_send) != (!d_recv) || ((uintptr_t)d_send & 255) || ((uintptr_t)d_recv & 255)) return BB_ERR_ARG;
    CK(cudaSetDevice(s->e->device));
    CK(cudaDeviceSynchronize());
    s->x_send = (uint8_t*)d_send; s->x_recv = (uint8_t*)d_recv;
    return BB_OK;
}
size_t bb_shard_exchange_bytes(const bb_shard* s) { return s ? s->reg_size * s->nranks * 2 : 0; }
uint32_t bb_shard_exchange_set(const bb_shard* s) { return s ? (s->epoch & 1) : 0; }
// geometry of one region: [0] bytes per region, [1] capacity in queries, [2] byte offset of the u32 offset array (cap + 1
// entries), [3] of the u32 ingress-index array (cap entries), [4] of the packed packet bytes; the first 16 bytes are the
// header {count, packet bytes, epoch, sender overflow flag}
void bb_shard_region_layout(const bb_shard* s, uint64_t out[5]) {
    if (!s || !out) return;
    out[0] = s->reg_size; out[1] = s->cap_q; out[2] = bbk::region_off_array(s->cap_q); out[3] = bbk::region_qidx_array(s->cap_q); out[4] = bbk::region_bytes(s->cap_q);
}

// Ingress: route every query of a device-resident batch to its owner and push it there.
int bb_shard_route_push(bb_shard* s, const uint8_t* d_pkts, const uint32_t* d_pkt_off, uint32_t n, uint32_t qidx_base, void* stream) {
    if (!s || n > s->max_batch || ((uintptr_t)d_pkts & 15)) return BB_ERR_ARG;
    for (uint32_t r = 0; r < s->nranks; r++) if (!s->x_send && !s->peer_recv[r]) return BB_ERR_ARG;
    bb_engine* e = s->e;
    bbk::PushParams A; memset(&A, 0, sizeof A);
    A.P.pkts = d_pkts; A.P.pkt_off = d_pkt_off; A.P.n = n; A.P.eng = e->d_const; A.P.ready = 1;
    A.P.suffix_len = e->hconst.suffix_len; A.P.soa_len = e->hconst.soa_len; A.P.recursion = e->hconst.recursion; A.P.lean_ok = e->hconst.lean_ok;
    A.P.route = 1; A.P.nranks = s->nranks; A.P.rank = s->rank; A.P.table = e->d_table; A.P.mask = e->mask; A.P.arena = e->d_arena;
    A.epoch = ++s->epoch;
    const size_t set = (size_t)(s->epoch & 1) * s->nranks;
    for (uint32_t r = 0; r < s->nranks; r++)
        A.region[r] = s->x_send ? s->x_send + (set + r) * s->reg_size                 // local send region for destination r
                                : s->peer_recv[r] + (set + s->rank) * s->reg_size;    // region (this rank -> r) in r's HBM
    A.cap_q = s->cap_q; A.cap_b = s->cap_b; A.cursor = s->cursor; A.done = s->done; A.err = s->err;
    A.qidx_base = qidx_base; A.P.stage_log = e->stage_log;
    // n == 0 still publishes empty region headers (one block, no queries)
    const uint32_t grid = n ? (n + bbk::T - 1) / bbk::T : 1;
    bbk::route_push_kernel<<<grid, bbk::T, 0, (cudaStream_t)stream>>>(A);
    CK(cudaGetLastError());
    e->launches++;
    return BB_OK;
}

// Owner: resolve the nranks receive regions (after the caller's cross-rank barrier), one launch
// per region on forked streams that join back into `stream`.
int bb_shard_resolve(bb_shard* s, uint64_t seed, int wait_for_peers, void* stream) {
    if (!s) return BB_ERR_ARG;
    bb_engine* e = s->e;
    cudaStream_t main = (cudaStream_t)stream;
    if (wait_for_peers) {
        bbk::wait_regions_kernel<<<1, 32, 0, main>>>(s->recv_base() + (size_t)(s->epoch & 1) * s->nranks * s->reg_size, s->reg_size, s->nranks,
                                                      s->epoch, s->err);
        CK(cudaGetLastError());
    }
    uint8_t* reg = s->recv_base() + (size_t)(s->epoch & 1) * s->nranks * s->reg_size;   // region 0 of the set just pushed
    bbk::Params P; memset(&P, 0, sizeof P);
    P.pkts = reg + bbk::region_bytes(s->cap_q); P.pkt_off = (const uint32_t*)(reg + bbk::region_off_array(s->cap_q));
    P.n = 0; P.n_dev = (const uint32_t*)reg; P.qidx_map = (const uint32_t*)(reg + bbk::region_qidx_array(s->cap_q));
    P.seed = seed; P.qidx_base = 0;
    P.out = s->d_out; P.out_cap = s->out_cap; P.out_off = (uint32_t*)s->d_out_off; P.out_len = (uint16_t*)s->d_out_len;
    P.status = s->d_status; P.miss_idx = (uint32_t*)s->d_miss; P.totals = (uint32_t*)s->d_totals;
    P.err_in = s->err;
    if (s->host) {                                   // results straight into the pinned mirrors (zero-copy)
        P.out = s->h_out; P.out_off = (uint32_t*)s->h_out_off; P.out_len = (uint16_t*)s->h_out_len; P.status = s->h_status;
        P.miss_idx = (uint32_t*)s->h_miss; P.totals = (uint32_t*)s->h_totals; P.qidx_out = (uint32_t*)s->h_qidx;
        P.bounce = s->d_out;                         // tiles too large to stage assemble on the device first
    }
    P.table = e->d_table; P.mask = e->mask; P.arena = e->d_arena; P.ready = e->ready && e->d_table; P.eng = e->d_const;
    P.suffix_len = e->hconst.suffix_len; P.soa_len = e->hconst.soa_len; P.recursion = e->hconst.recursion; P.lean_ok = e->hconst.lean_ok;
    P.ntiles = (s->cap_q + bbk::T - 1) / bbk::T; P.ntiles_cap = e->max_tiles;
    P.desc = (unsigned long long*)s->d_desc; P.counter = (uint32_t*)((unsigned long long*)s->d_desc + e->max_tiles + 1);
    P.epoch = (uint32_t)(++e->epoch); P.stage_log = nullptr; P.route = 0; P.nranks = s->nranks; P.rank = s->rank;
    P.regions = 1; P.in_stride = s->reg_size; P.out_stride = s->out_stride; P.off_stride = s->off_stride; P.len_stride = s->len_stride;
    P.status_stride = s->status_stride; P.miss_stride = s->miss_stride; P.totals_stride = s->totals_stride; P.desc_stride = s->desc_stride;
    const dim3 grid(P.ntiles, s->nranks);
    if (e->ordered) bbk::resolve_kernel<true, true, false><<<grid, bbk::T, 0, main>>>(P);
    else bbk::resolve_kernel<false, true, false><<<grid, bbk::T, 0, main>>>(P);
    CK(cudaGetLastError());
    s->resolve_epoch = P.epoch;
    e->launches++;
    return BB_OK;
}

// Pinned host mirrors of the per-region result set: from now on bb_shard_resolve writes responses,
// offsets, lengths, statuses, ingress indices, miss lists and totals straight into host memory
// (no copies, no size round trip), and bb_shard_results hands out pointers into them.
int bb_shard_host_results(bb_shard* s, int enable) {
    if (!s) return BB_ERR_ARG;
    CK(cudaSetDevice(s->e->device));
    if (enable && !s->h_out) {
        const unsigned fl = cudaHostAllocPortable | cudaHostAllocMapped;
        const size_t R = s->nranks;
        CK(cudaHostAlloc((void**)&s->h_out, s->out_stride * R, fl)); CK(cudaHostAlloc((void**)&s->h_out_off, s->off_stride * R, fl));
        CK(cudaHostAlloc((void**)&s->h_out_len, s->len_stride * R, fl)); CK(cudaHostAlloc((void**)&s->h_status, s->status_stride * R, fl));
        CK(cudaHostAlloc((void**)&s->h_miss, s->miss_stride * R, fl)); CK(cudaHostAlloc((void**)&s->h_totals, s->totals_stride * R, fl));
        CK(cudaHostAlloc((void**)&s->h_qidx, s->off_stride * R, fl));
        memset(s->h_totals, 0, s->totals_stride * R);
    }
    CK(cudaDeviceSynchronize());                     // resolves in flight finish with the old destination
    s->host = enable != 0;
    return BB_OK;
}

// Region `src` of the last bb_shard_resolve, in the host mirrors.  The caller has waited for the work
// it enqueued on the resolve's stream (event or stream synchronize); BB_ERR_ARG if that resolve has
// not finished writing this region.  The pointers stay valid until the next resolve on this shard.
int bb_shard_results(bb_shard* s, uint32_t src, const uint8_t** out, const uint32_t** out_off, const uint16_t** out_len,
                     const uint8_t** status, const uint32_t** qidx, const uint32_t** miss_idx,
                     uint32_t* n_out, uint32_t* n_miss, uint32_t* total_out) {
    if (!s || src >= s->nranks || !s->host || !s->resolve_epoch) return BB_ERR_ARG;
    const volatile uint32_t* tot = (const volatile uint32_t*)(s->h_totals + src * s->totals_stride);
    if (tot[3] != s->resolve_epoch) return BB_ERR_ARG;
    if (tot[6] == 2) { g_cuda_err = "timed out waiting for a peer rank's push"; return BB_ERR_CUDA; }
    if (tot[5] || tot[2] == s->resolve_epoch) return BB_ERR_CAPACITY;      // a sender overflowed the region / responses overflowed out
    const uint32_t n = tot[4];
    *n_out = n; *n_miss = n ? tot[1] : 0; *total_out = n ? tot[0] : 0;
    *out = s->h_out + src * s->out_stride; *out_off = (const uint32_t*)(s->h_out_off + src * s->off_stride);
    *out_len = (const uint16_t*)(s->h_out_len + src * s->len_stride); *status = s->h_status + src * s->status_stride;
    *qidx = (const uint32_t*)(s->h_qidx + src * s->off_stride); *miss_idx = (const uint32_t*)(s->h_miss + src * s->miss_stride);
    return BB_OK;
}

// Results of region `src` to host memory (synchronous).  qidx[i] is the index the query had in
// rank src's ingress numbering (qidx_base + position).  Returns the region's query count in *n_out.
int bb_shard_fetch(bb_shard* s, uint32_t src, uint8_t* out, uint32_t out_cap, uint32_t* out_off, uint16_t* out_len,
                   uint8_t* status, uint32_t* qidx, uint32_t* miss_idx, uint32_t* n_out, uint32_t* n_miss, uint32_t* total_out) {
    if (!s || src >= s->nranks || s->host) return BB_ERR_ARG;       // host mirrors on: use bb_shard_results
    CK(cudaSetDevice(s->e->device));
    uint8_t* reg = s->recv_base() + ((size_t)(s->epoch & 1) * s->nranks + src) * s->reg_size;
    uint32_t hdr[4], tot[4];
    CK(cudaMemcpy(hdr, reg, 16, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(tot, s->d_totals + src * s->totals_stride, 16, cudaMemcpyDeviceToHost));
    if (hdr[3]) return BB_ERR_CAPACITY;                          // a sender overflowed this region
    { uint32_t werr = 0; CK(cudaMemcpy(&werr, s->err, 4, cudaMemcpyDeviceToHost)); if (werr == 2) { g_cuda_err = "timed out waiting for a peer rank's push"; return BB_ERR_CUDA; } }
    const uint32_t n = hdr[0];
    *n_out = n; *n_miss = n ? tot[1] : 0; *total_out = n ? tot[0] : 0;
    if (!n) return BB_OK;
    if (tot[2] == s->resolve_epoch || tot[0] > s->out_cap || tot[0] > out_cap) return BB_ERR_CAPACITY;   // the region's responses overflowed the shard's buffer / the caller's
    CK(cudaMemcpy(out, s->d_out + src * s->out_stride, tot[0], cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(out_off, s->d_out_off + src * s->off_stride, ((size_t)n + 1) * 4, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(out_len, s->d_out_len + src * s->len_stride, (size_t)n * 2, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(status, s->d_status + src * s->status_stride, n, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(qidx, reg + bbk::region_qidx_array(s->cap_q), (size_t)n * 4, cudaMemcpyDeviceToHost));
    if (tot[1]) CK(cudaMemcpy(miss_idx, s->d_miss + src * s->miss_stride, (size_t)tot[1] * 4, cudaMemcpyDeviceToHost));
    return BB_OK;
}

}  // extern "C"
