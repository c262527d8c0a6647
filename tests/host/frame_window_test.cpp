// Host-side driver of the compressor's Window_Descriptor rule (frame_window_log and write_frame_header in
// zstd-rs_b200/csrc/encode.cuh), read back with the decoder's parser (parse_frame_header in zstd-rs_b200/csrc/framing.cuh).
// Arguments: a list of "<content size>:<window_log>".  Prints one line per case: "<header hex> <frame_window_log> <parse status>
// <window size>"; tests/test_cldm_model.py checks it against tests/cparse.py.
#include <cinttypes>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include "../../zstd-rs_b200/csrc/encode.cuh"
#include "../../zstd-rs_b200/csrc/framing.cuh"
using namespace b200z;

int main(int argc, char **argv) {
    for (int i = 1; i < argc; i++) {
        char *p = argv[i];
        const uint64_t n = strtoull(p, &p, 10);
        const uint32_t wl = (uint32_t)strtoul(p + 1, &p, 10);
        uint8_t hdr[32] = {0};
        const uint32_t w = frame_window_log(n, wl);
        const uint32_t len = write_frame_header(hdr, n, true, 0, w);
        FrameHeader h;
        uint32_t skip = 0;
        size_t consumed = 0;
        int st = parse_frame_header(hdr, len, h, skip, consumed);
        uint64_t ws = 0;
        if (!st) st = frame_window_size(h, ws);
        for (uint32_t k = 0; k < len; k++) printf("%02x", hdr[k]);
        printf(" %u %d %" PRIu64 "\n", w, st, ws);
    }
    return 0;
}
