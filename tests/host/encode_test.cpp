// Host-side driver of zstd-rs_b200/csrc/encode.cuh (the block encoder k_cenc runs on the GPU), for tests/seqcraft.py.
//   encode_test [--ov] IN OUT   IN = u32 nlit, nlit literal bytes, u32 nseq, nseq x {u32 ll, ml, of}
//                               OUT = the content of a Compressed block for them
// With --ov the third field is the zstd Offset_Value itself (1-3 are repeat codes): the encoder writes of + 3 with code
// flog2(of + 3), so passing ov - 3 (mod 2^32) emits exactly ov.
// It checks what the format needs of the tables -- Huffman lengths <= 11 with a complete code, FSE counts summing to 2^log --
// and prints "ok <content size> <huffman literals 0/1> <LL mode> <OF mode> <ML mode>".
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>
#include "../../zstd-rs_b200/csrc/encode.cuh"
using namespace b200z;

#define CHECK(c) do { if (!(c)) { printf("FAIL %s:%d %s\n", __FILE__, __LINE__, #c); return 1; } } while (0)

int main(int argc, char **argv) {
    const bool ov = argc == 4 && !strcmp(argv[1], "--ov");
    if (argc != 3 && !ov) return 2;
    argv += ov ? 1 : 0;
    FILE *f = fopen(argv[1], "rb");
    if (!f) return 2;
    uint32_t nlit = 0, nseq = 0;
    if (fread(&nlit, 4, 1, f) != 1) return 2;
    std::vector<uint8_t> lits(nlit + 1);
    if (fread(lits.data(), 1, nlit, f) != nlit || fread(&nseq, 4, 1, f) != 1) return 2;
    std::vector<SeqRec> seqs(nseq + 1);
    if (fread(seqs.data(), sizeof(SeqRec), nseq, f) != nseq) return 2;
    fclose(f);
    if (ov)
        for (uint32_t i = 0; i < nseq; i++) seqs[i].of -= 3;
    static EncScratch s;
    const uint32_t cap = 4 * ENC_BLOCK;
    std::vector<uint8_t> out(cap);
    const uint32_t n = encode_block(s, lits.data(), nlit, seqs.data(), nseq, out.data(), cap, 0, 1);
    CHECK(n <= cap);
    if (s.use_huf) {
        uint32_t kraft = 0, maxb = 0;
        for (int i = 0; i < 256; i++) {
            CHECK(s.huf_len[i] <= ENC_HUF_MAX_BITS);
            CHECK((s.huf_len[i] != 0) == (s.lit_cnt[i] != 0));
            if (s.huf_len[i]) kraft += 1u << (ENC_HUF_MAX_BITS - s.huf_len[i]);
            if (s.huf_len[i] > maxb) maxb = s.huf_len[i];
        }
        CHECK(kraft == 1u << ENC_HUF_MAX_BITS);
    }
    uint32_t modes[3] = {0, 0, 0};
    if (nseq) {
        for (uint32_t t = 0; t < 3; t++) {
            modes[t] = s.mode[t];
            if (s.mode[t] != 2) continue;
            CHECK(s.ct[t].log >= 5 && s.ct[t].log <= enc_max_log(t));
            int32_t sum = 0;
            for (uint32_t c = 0; c <= s.maxsym[t]; c++) {
                CHECK((s.norm[t][c] != 0) == (s.cnt[t][c] != 0));
                sum += s.norm[t][c] < 0 ? 1 : s.norm[t][c];
            }
            CHECK(sum == 1 << s.ct[t].log);
        }
    }
    f = fopen(argv[2], "wb");
    if (!f || fwrite(out.data(), 1, n, f) != n) return 2;
    fclose(f);
    printf("ok %u %u %u %u %u\n", n, s.use_huf, modes[0], modes[1], modes[2]);
    return 0;
}
