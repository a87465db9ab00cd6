// CPU emulation of the relay kernel's per-relay work: the SAME device source (binder_b200/csrc/relay_device.cuh, with
// the query decode() and byte emitter of resolve_device.cuh) compiled for the host through tests/native/cuda_shim.h.
// Every relay's query and upstream are copied into buffers of exactly their length, and every reply is emitted into a
// buffer of exactly its sized length, so that a build with -fsanitize=address,undefined catches any read past a packet
// or any write past a reply.  The cooperative kernel body (staging, scan, placement, flush) is covered by the -m gpu
// tests.  Test infrastructure, not product (tests/test_relay.py).
//
//   emu_relay IN OUT    IN  = u32 n, u32 flags, u32 q_off[n+1], u32 up_off[n+1], query bytes, upstream bytes
//                       OUT = u32 out_off[n+1], u8 status[n], reply bytes (packed in order)
#include "cuda_shim.h"
#include "../../binder_b200/csrc/zone_image.h"
#include "../../include/binder_b200.h"
namespace bbk { thread_local unsigned long long bb_emu_lean_count = 0, bb_emu_general_count = 0; }
#include "../../binder_b200/csrc/resolve_device.cuh"
#include "../../binder_b200/csrc/relay_device.cuh"

#include <cstdio>
#include <vector>

thread_local uint8_t* bb_emu_smem = nullptr;

static bool read_all(const char* path, std::vector<uint8_t>& buf) {
    FILE* f = fopen(path, "rb");
    if (!f) return false;
    uint8_t tmp[1 << 16];
    size_t k;
    while ((k = fread(tmp, 1, sizeof tmp, f)) > 0) buf.insert(buf.end(), tmp, tmp + k);
    fclose(f);
    return true;
}

int main(int argc, char** argv) {
    std::vector<uint8_t> in;
    if (argc != 3 || !read_all(argv[1], in) || in.size() < 8) { fprintf(stderr, "usage: emu_relay IN OUT\n"); return 2; }
    uint32_t n, flags;
    memcpy(&n, in.data(), 4); memcpy(&flags, in.data() + 4, 4);
    const size_t hdr = 8 + 8 * ((size_t)n + 1);
    if (in.size() < hdr) return 2;
    std::vector<uint32_t> q_off(n + 1), up_off(n + 1);
    memcpy(q_off.data(), in.data() + 8, 4 * ((size_t)n + 1));
    memcpy(up_off.data(), in.data() + 8 + 4 * ((size_t)n + 1), 4 * ((size_t)n + 1));
    const uint8_t* qb = in.data() + hdr;
    const uint8_t* ub = qb + q_off[n];
    if (in.size() < hdr + q_off[n] + up_off[n]) return 2;
    std::vector<uint32_t> out_off(n + 1, 0);
    std::vector<uint8_t> status(n), out;
    for (uint32_t i = 0; i < n; i++) {
        std::vector<uint8_t> q(qb + q_off[i], qb + q_off[i + 1]), u(ub + up_off[i], ub + up_off[i + 1]);
        bbk::Relay R;
        bbk::relay_size(q.data(), (uint32_t)q.size(), u.data(), (uint32_t)u.size(), (flags & BB_BATCH_TCP) != 0, R);
        status[i] = (uint8_t)R.status;
        out_off[i] = (uint32_t)out.size();
        if (R.status != bbk::ST_ANSWERED) continue;
        std::vector<uint8_t> reply(R.rlen);
        bbk::relay_emit(q.data(), u.data(), (uint32_t)u.size(), R, reply.data());
        out.insert(out.end(), reply.begin(), reply.end());
    }
    out_off[n] = (uint32_t)out.size();
    FILE* f = fopen(argv[2], "wb");
    if (!f) return 2;
    fwrite(out_off.data(), 4, n + 1, f);
    fwrite(status.data(), 1, n, f);
    fwrite(out.data(), 1, out.size(), f);
    fclose(f);
    printf("OK %u\n", n);
    return 0;
}
