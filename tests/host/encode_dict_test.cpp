// Host-side driver of encode_block with a formatted dictionary's tables (zstd-rs_b200/csrc/encode.cuh), for
// tests/test_encode_dict_host.py.
//   encode_dict_test DICT IN OUT   DICT = a zstd-format dictionary; IN / OUT as encode_test (u32 nlit, literals, u32 nseq,
//                                  nseq x {u32 ll, ml, of}; OUT = the content of a Compressed block, the frame's first block)
//   encode_dict_test DICT          prints the dictionary's tables as the encoder sees them: "tables <bytes without a Huffman code>
//                                  <LL codes with count 0> <OF ...> <ML ...>", each a comma-separated list ("-" when empty)
// The dictionary is parsed with the decoder's readers (tables.cuh) and turned into an EncDict by enc_dict_build, as
// b200z_dict_create and the batch compressor do.  Prints "ok <content size> <literals: 0 raw, 1 own Huffman, 3 Treeless>
// <LL mode> <OF mode> <ML mode>".
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>
#include "../../zstd-rs_b200/csrc/encode.cuh"
using namespace b200z;

static bool load_dict(const char *path, EncDict &d) {
    FILE *f = fopen(path, "rb");
    if (!f) return false;
    std::vector<uint8_t> raw(1 << 22);
    const size_t len = fread(raw.data(), 1, raw.size(), f);
    fclose(f);
    if (len < 8 || raw[0] != 0x37 || raw[1] != 0xA4 || raw[2] != 0x30 || raw[3] != 0xEC) return false;
    const uint8_t *t = raw.data() + 8;
    uint32_t tl = (uint32_t)len - 8, used = 0;
    static uint8_t weights[260];
    uint32_t nweights = 0;
    if (huf_read_weights(t, tl, weights, nweights, used) || used > tl) return false;
    t += used; tl -= used;
    static int16_t probs[3][256];
    uint32_t nprobs[3], logs[3];
    const uint32_t order[3] = {ENC_OF, ENC_ML, ENC_LL}, max_log[3] = {8, 9, 9}, max_sym[3] = {31, 52, 35};
    for (int i = 0; i < 3; i++) {
        const uint32_t e = order[i];
        if (fse_read_probabilities(t, tl, max_log[i], max_sym[i], probs[e], nprobs[e], logs[e], used) || used > tl) return false;
        t += used; tl -= used;
    }
    const int16_t *p[3] = {probs[0], probs[1], probs[2]};
    enc_dict_build(weights, nweights, p, nprobs, logs, d);
    return true;
}

static std::string list(const std::vector<uint32_t> &v) {
    std::string s;
    for (uint32_t x : v) s += (s.empty() ? "" : ",") + std::to_string(x);
    return s.empty() ? "-" : s;
}

int main(int argc, char **argv) {
    static EncDict dt;
    if (argc < 2 || !load_dict(argv[1], dt)) return 2;
    if (argc == 2) {
        std::vector<uint32_t> nolit, nocode[3];
        for (uint32_t i = 0; i < 256; i++) if (!dt.huf_len[i]) nolit.push_back(i);
        for (uint32_t t = 0; t < 3; t++)
            for (uint32_t c = 0; c <= enc_max_sym(t); c++) if (!dt.norm[t][c]) nocode[t].push_back(c);
        printf("tables %s %s %s %s\n", list(nolit).c_str(), list(nocode[ENC_LL]).c_str(), list(nocode[ENC_OF]).c_str(), list(nocode[ENC_ML]).c_str());
        return 0;
    }
    if (argc != 4) return 2;
    FILE *f = fopen(argv[2], "rb");
    if (!f) return 2;
    uint32_t nlit = 0, nseq = 0;
    if (fread(&nlit, 4, 1, f) != 1) return 2;
    std::vector<uint8_t> lits(nlit + 1);
    if (fread(lits.data(), 1, nlit, f) != nlit || fread(&nseq, 4, 1, f) != 1) return 2;
    std::vector<SeqRec> seqs(nseq + 1);
    if (fread(seqs.data(), sizeof(SeqRec), nseq, f) != nseq) return 2;
    fclose(f);
    static EncScratch s;
    const uint32_t cap = 4 * ENC_BLOCK;
    std::vector<uint8_t> out(cap);
    const uint32_t n = encode_block(s, lits.data(), nlit, seqs.data(), nseq, out.data(), cap, 0, 1, &dt);
    if (n > cap) return 3;
    f = fopen(argv[3], "wb");
    if (!f || fwrite(out.data(), 1, n, f) != n) return 2;
    fclose(f);
    printf("ok %u %u %u %u %u\n", n, s.use_dict ? 3u : s.use_huf, nseq ? s.mode[0] : 0u, nseq ? s.mode[1] : 0u, nseq ? s.mode[2] : 0u);
    return 0;
}
