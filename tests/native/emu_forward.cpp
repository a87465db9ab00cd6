// CPU emulation of the forward and match kernels' per-miss and per-response work: the SAME device source
// (binder_b200/csrc/forward_device.cuh, with decode() and the pre-filter scan of resolve_device.cuh) compiled for the host
// through tests/native/cuda_shim.h.  Every miss and every received datagram is copied into a buffer of exactly its
// length, and every upstream query is written into a buffer of exactly its length, so that a build with
// -fsanitize=address,undefined catches any read past a datagram or write past a query.  The cooperative parts of the
// kernels (staging, scans, grouping, the earliest-arrival atomic) are covered by the -m gpu tests; here the earliest
// accepted response per miss is kept by a loop in arrival order.  Test infrastructure, not product (tests/test_forward_emu.py).
//
//   emu_forward IN OUT
//   IN  = u32 n_dc, n_dc x (u32 len, bytes), u32 region_len, region bytes, u32 n_up, u32 ip[n_up], u16 port[n_up],
//         u8 dc[n_up], u64 key, u32 n, u32 off[n+1], miss bytes, u32 n_resp, u32 resp_off[n_resp+1], u32 src_ip[n_resp],
//         u16 src_port[n_resp], response bytes
//   OUT = u8 route[n], u32 uq_off[n+1] (miss order), upstream query bytes, u32 winner[n] (response index or 0xFFFFFFFF)
#include "cuda_shim.h"
#include "../../binder_b200/csrc/zone_image.h"
#include "../../include/binder_b200.h"
namespace bbk { thread_local unsigned long long bb_emu_lean_count = 0, bb_emu_general_count = 0; }
#include "../../binder_b200/csrc/resolve_device.cuh"
#include "../../binder_b200/csrc/forward_device.cuh"

#include <cstdio>
#include <string>
#include <vector>

thread_local uint8_t* bb_emu_smem = nullptr;

struct Reader {
    std::vector<uint8_t> b; size_t pos = 0; bool ok = true;
    template <class V> V get() { V v{}; if (pos + sizeof v > b.size()) { ok = false; return v; } memcpy(&v, b.data() + pos, sizeof v); pos += sizeof v; return v; }
    template <class V> std::vector<V> arr(size_t n) { std::vector<V> v(n); for (auto& x : v) x = get<V>(); return v; }
    std::vector<uint8_t> bytes(size_t n) { if (pos + n > b.size()) { ok = false; return {}; } std::vector<uint8_t> v(b.begin() + pos, b.begin() + pos + n); pos += n; return v; }
};

int main(int argc, char** argv) {
    Reader r;
    FILE* f = argc == 3 ? fopen(argv[1], "rb") : nullptr;
    if (!f) { fprintf(stderr, "usage: emu_forward IN OUT\n"); return 2; }
    uint8_t tmp[1 << 16]; size_t k;
    while ((k = fread(tmp, 1, sizeof tmp, f)) > 0) r.b.insert(r.b.end(), tmp, tmp + k);
    fclose(f);
    const uint32_t n_dc = r.get<uint32_t>();
    std::vector<std::string> names;
    for (uint32_t i = 0; i < n_dc && r.ok; i++) { const auto v = r.bytes(r.get<uint32_t>()); names.emplace_back(v.begin(), v.end()); }
    const auto reg = r.bytes(r.get<uint32_t>());
    const std::string region(reg.begin(), reg.end());
    const uint32_t n_up = r.get<uint32_t>();
    const auto ip = r.arr<uint32_t>(n_up); const auto port = r.arr<uint16_t>(n_up); const auto dc = r.arr<uint8_t>(n_up);
    const uint64_t key = r.get<uint64_t>();
    const uint32_t n = r.get<uint32_t>();
    const auto off = r.arr<uint32_t>((size_t)n + 1);
    const auto pk = r.bytes(r.ok ? off[n] : 0);
    const uint32_t n_resp = r.get<uint32_t>();
    const auto roff = r.arr<uint32_t>((size_t)n_resp + 1);
    const auto rip = r.arr<uint32_t>(n_resp); const auto rport = r.arr<uint16_t>(n_resp);
    const auto rb = r.bytes(r.ok ? roff[n_resp] : 0);
    if (!r.ok) { fprintf(stderr, "short input\n"); return 2; }

    bb::EngineConst* E = new bb::EngineConst();
    std::vector<const char*> np; for (auto& s : names) np.push_back(s.c_str());
    if (!bb::make_engine_const("example.com", true, *E) || !bb::set_recursion_filter_const(*E, region.c_str(), np.data(), n_dc, true) ||
        !bb::set_recursion_upstreams_const(*E, ip.data(), port.data(), dc.data(), n_up)) { fprintf(stderr, "bad table\n"); return 2; }
    const bbk::IdKey K = bbk::id_key_rounds(key);

    // forward, miss by miss
    std::vector<uint8_t> route(n), uq;
    std::vector<uint32_t> uq_off(n + 1, 0);
    std::vector<uint8_t> clients(pk);                 // the client queries packed in miss order (the forward kernel's copy)
    for (uint32_t j = 0; j < n; j++) {
        std::vector<uint8_t> q(pk.begin() + off[j], pk.begin() + off[j + 1]);
        route[j] = (uint8_t)bbk::RT_NONE;
        uq_off[j] = (uint32_t)uq.size();
        bbk::Res d;
        if (q.size() > 65535 || !bbk::decode(q.data(), (uint32_t)q.size(), d)) continue;
        route[j] = (uint8_t)bbk::fwd_route(E, q.data(), d);
        std::vector<uint8_t> msg(12 + d.qn_len + 4);
        bbk::fwd_emit(q.data(), d.qn_len, bbk::id_enc(K, j), msg.data());
        uq.insert(uq.end(), msg.begin(), msg.end());
    }
    uq_off[n] = (uint32_t)uq.size();
    // match, datagram by datagram in arrival order
    std::vector<uint32_t> win(n, bbk::NO_MATCH);
    for (uint32_t i = 0; i < n_resp; i++) {
        std::vector<uint8_t> u(rb.begin() + roff[i], rb.begin() + roff[i + 1]);
        const uint32_t j = bbk::match_one(E, K, u.data(), (uint32_t)u.size(), rip[i], rport[i], n, route.data(), clients.data(), off.data());
        if (j != bbk::NO_MATCH && win[j] == bbk::NO_MATCH) win[j] = i;
    }
    delete E;
    FILE* o = fopen(argv[2], "wb");
    if (!o) return 2;
    fwrite(route.data(), 1, n, o);
    fwrite(uq_off.data(), 4, (size_t)n + 1, o);
    fwrite(uq.data(), 1, uq.size(), o);
    fwrite(win.data(), 4, n, o);
    fclose(o);
    printf("OK %u %u\n", n, n_resp);
    return 0;
}
