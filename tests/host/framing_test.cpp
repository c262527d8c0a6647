// Host-side driver of the header parsers in zstd-rs_b200/csrc/framing.cuh (shared by the host planner and k_walk).  Reads one case
// per line from the file named by argv[1] and prints one result line per case; tests/test_host_units.py builds the cases and checks
// the results against the CPU oracle and tests/refwalk.py.
//   "F <hex>"  a source holding these bytes, read the way the frame decoder's reset reads it (frame_header_want: the magic number,
//              then the descriptor byte or a skippable frame's length, then the rest of the header), then parse_frame_header and the
//              checks reset applies after it (window size, default window limit, dictionary lookup with no dictionary).
//              Prints "<error> <bytes taken from the source>".
//   "S <hex>"  parse_section_headers on a Compressed block's content.
//              Prints "<status> <lit_type> <nstreams> <regen_size> <lit_comp_size> <lit_off> <nseq> <modes> <seq_off>".
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <vector>
#include "../../zstd-rs_b200/csrc/framing.cuh"
using namespace b200z;

int main(int argc, char **argv) {
    if (argc != 2) return 2;
    FILE *in = fopen(argv[1], "r");
    if (!in) return 2;
    static char line[1 << 19];   // a whole block (128 KiB) in hex
    while (fgets(line, sizeof line, in)) {
        std::vector<uint8_t> b;
        for (const char *q = line + 2; q[0] && q[1] && q[0] != '\n'; q += 2) {
            unsigned v;
            if (sscanf(q, "%2x", &v) != 1) return 2;
            b.push_back((uint8_t)v);
        }
        if (line[0] == 'F') {
            uint8_t buf[32];
            size_t have = 0;
            for (size_t want; (want = frame_header_want(buf, have)) > have;) {
                const size_t got = want < b.size() ? want : b.size();
                if (got > have) memcpy(buf + have, b.data() + have, got - have);
                have = got;
                if (have < want) break;
            }
            FrameHeader h;
            uint32_t skip = 0;
            size_t consumed = 0;
            int e = parse_frame_header(buf, have, h, skip, consumed);
            uint64_t window = 0;
            if (!e) e = frame_window_size(h, window);
            if (!e && window > B200Z_DEFAULT_MAX_WINDOW_SIZE) e = B200Z_ERR_WINDOW_SIZE_TOO_BIG;
            if (!e && h.has_dict_id) e = B200Z_ERR_DICT_NOT_PROVIDED;
            if (consumed != have || (!e && h.header_size != have)) { printf("consumed %zu, header %u, read %zu\n", consumed, h.header_size, have); return 1; }
            printf("%d %zu\n", e, have);
        } else if (line[0] == 'S') {
            const SectionHeaders s = parse_section_headers(b.data(), (uint32_t)b.size());
            printf("%u %u %u %u %u %u %u %u %u\n", s.status, s.lit_type, s.nstreams, s.regen_size, s.lit_comp_size, s.lit_off, s.nseq, s.modes, s.seq_off);
        } else {
            return 2;
        }
    }
    return 0;
}
