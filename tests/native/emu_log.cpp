// CPU emulation of the log kernel's per-response work: the SAME device source (binder_b200/csrc/log_device.cuh, with
// relay_device.cuh's name and RR decode and resolve_device.cuh's helpers) compiled for the host through
// tests/native/cuda_shim.h.  Every response is copied into a buffer of exactly its length, and every record is emitted
// into a buffer of exactly its sized length, so that a build with -fsanitize=address,undefined catches any read past a
// response or any write past a record.  The cooperative kernel body (staging, scan, placement, flush) is covered by the
// -m gpu tests.  Test infrastructure, not product (tests/test_query_log.py).
//
//   emu_log IN OUT    IN  = u32 n, u32 resp_bytes, u32 sl, u8 sfx[sl], u32 out_off[n], u16 out_len[n], u8 status[n],
//                           u8 resp[resp_bytes]
//                     OUT = u32 log_len[n], u32 head_len[n], u32 summary[n], record bytes (packed in order)
#include "cuda_shim.h"
#include "../../binder_b200/csrc/zone_image.h"
#include "../../include/binder_b200.h"
namespace bbk { thread_local unsigned long long bb_emu_lean_count = 0, bb_emu_general_count = 0; }
#include "../../binder_b200/csrc/resolve_device.cuh"
#include "../../binder_b200/csrc/relay_device.cuh"
#include "../../binder_b200/csrc/log_device.cuh"

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
    if (argc != 3 || !read_all(argv[1], in) || in.size() < 12) { fprintf(stderr, "usage: emu_log IN OUT\n"); return 2; }
    uint32_t n, rb, sl;
    memcpy(&n, in.data(), 4); memcpy(&rb, in.data() + 4, 4); memcpy(&sl, in.data() + 8, 4);
    const size_t at_off = 12 + (size_t)sl, at_len = at_off + 4 * (size_t)n, at_st = at_len + 2 * (size_t)n, at_resp = at_st + n;
    if (sl > 256 || in.size() != at_resp + rb) return 2;
    const std::vector<uint8_t> sfx(in.begin() + 12, in.begin() + at_off);
    std::vector<uint32_t> out_off(n), log_len(n), head_len(n), summary(n);
    std::vector<uint16_t> out_len(n);
    memcpy(out_off.data(), in.data() + at_off, 4 * (size_t)n);
    memcpy(out_len.data(), in.data() + at_len, 2 * (size_t)n);
    const uint8_t* status = in.data() + at_st;
    const uint8_t* resp = in.data() + at_resp;
    std::vector<uint8_t> text;
    for (uint32_t i = 0; i < n; i++) {
        const uint32_t o = out_off[i], l = out_len[i];
        if (status[i] != bbk::ST_ANSWERED) continue;
        if (o > rb || l > rb - o) { summary[i] = bbk::LOG_BAD; continue; }      // as log_kernel
        const std::vector<uint8_t> u(resp + o, resp + o + l);
        bbk::Txt t{ nullptr, 0 };
        uint32_t hl = 0;
        summary[i] = bbk::log_record(u.data(), l, sfx.data(), sl, t, hl);
        if (summary[i] & bbk::LOG_BAD) continue;
        std::vector<uint8_t> rec(t.n);
        bbk::Txt w{ rec.data(), 0 };
        uint32_t hl2 = 0;
        bbk::log_record(u.data(), l, sfx.data(), sl, w, hl2);
        if (w.n != t.n || hl2 != hl) { fprintf(stderr, "record %u: sized %u/%u, emitted %u/%u\n", i, t.n, hl, w.n, hl2); return 3; }
        log_len[i] = t.n; head_len[i] = hl;
        text.insert(text.end(), rec.begin(), rec.end());
    }
    FILE* f = fopen(argv[2], "wb");
    if (!f) return 2;
    fwrite(log_len.data(), 4, n, f);
    fwrite(head_len.data(), 4, n, f);
    fwrite(summary.data(), 4, n, f);
    fwrite(text.data(), 1, text.size(), f);
    fclose(f);
    printf("OK %u\n", n);
    return 0;
}
