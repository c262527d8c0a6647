// Host-side driver of the compressor's frame header writer (write_frame_header in zstd-rs_b200/csrc/encode.cuh), read back with the
// decoder's parser (parse_frame_header in zstd-rs_b200/csrc/framing.cuh).  Arguments: a list of "<content size>:<dictionary id>:<checksum 0/1>".
// Prints one line per case: "<header hex> <frame_header_size> <parse status> <has_dict_id> <dict_id> <frame_content_size>
// <checksum flag> <window descriptor> <header_size>"; tests/test_frame_header_dict.py checks it against a Python writer.
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
        const uint32_t id = (uint32_t)strtoul(p + 1, &p, 10);
        const bool checksum = strtoul(p + 1, &p, 10) != 0;
        uint8_t hdr[32] = {0};
        const uint32_t len = write_frame_header(hdr, n, checksum, id);
        FrameHeader h;
        uint32_t skip = 0;
        size_t consumed = 0;
        const int st = parse_frame_header(hdr, len, h, skip, consumed);
        for (uint32_t k = 0; k < len; k++) printf("%02x", hdr[k]);
        printf(" %u %d %d %u %" PRIu64 " %d %u %u\n", frame_header_size(n, id), st, h.has_dict_id ? 1 : 0, h.dict_id, h.frame_content_size,
               h.content_checksum() ? 1 : 0, h.window_descriptor, h.header_size);
    }
    return 0;
}
