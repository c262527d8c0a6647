#!/usr/bin/env python3
"""Generate tests/golden/ from the reference's own golden vectors (run in the build container only).

The reference (KillingSpark/zstd-rs @ eb7e03cc) is Rust and cannot be executed here, so the vectors are the
ones its own tests assert on (SURVEY.md section 8c):
  * ruzstd/decodecorpus_files/*.zst + originals   (tests/decode_corpus.rs)
  * ruzstd/dict_tests/{dictionary,files/*}        (tests/dict_test.rs)
  * ruzstd/test_fixtures/*.zst                    (tests/mod.rs:576-741; plaintexts generated in code)
  * ruzstd/fuzz/artifacts/*/*                     (tests/fuzz_regressions.rs, fse/mod.rs, huff0/mod.rs)
Compressed inputs are copied verbatim (they are test DATA, not source); expected plaintexts are recorded as
size + SHA-256 + XXH64-low32 in manifest.json, and the corpus originals as SHA-256 digests of every 64 KiB chunk in
decodecorpus_originals.json, so the repo stays small.  Every test reads tests/golden/ only.

    python tests/golden/make_golden.py <path to the ruzstd/ directory of a zstd-rs checkout>
"""
import hashlib, json, os, shutil, sys

REF = sys.argv[1] if len(sys.argv) > 1 else "ruzstd"
CHUNK = 64 << 10
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", ".."))


def sha(b):
    return hashlib.sha256(b).hexdigest()


def main():
    from oracle.oracle import xxh64
    man = {"source": "KillingSpark/zstd-rs eb7e03cc1b15705b94b93249ff7b05c4fc2c98b3", "corpus": {}, "dict": {}, "fixtures": {}, "fuzz": {}}
    chunks = {"chunk_bytes": CHUNK, "files": {}}
    # corpus
    dst = os.path.join(HERE, "decodecorpus"); os.makedirs(dst, exist_ok=True)
    for f in sorted(os.listdir(f"{REF}/decodecorpus_files")):
        if not f.endswith(".zst"):
            continue
        shutil.copyfile(f"{REF}/decodecorpus_files/{f}", f"{dst}/{f}")
        orig = open(f"{REF}/decodecorpus_files/{f[:-4]}", "rb").read()
        chunks["files"][f] = [sha(orig[i:i + CHUNK]) for i in range(0, max(len(orig), 1), CHUNK)]
        man["corpus"][f] = {"size": len(orig), "sha256": sha(orig), "xxh64_low32": xxh64(orig) & 0xFFFFFFFF,
                            "compressed_size": os.path.getsize(f"{dst}/{f}")}
    # dict tests
    dst = os.path.join(HERE, "dict_tests", "files"); os.makedirs(dst, exist_ok=True)
    shutil.copyfile(f"{REF}/dict_tests/dictionary", os.path.join(HERE, "dict_tests", "dictionary"))
    for f in sorted(os.listdir(f"{REF}/dict_tests/files")):
        if not f.endswith(".zst"):
            continue
        shutil.copyfile(f"{REF}/dict_tests/files/{f}", f"{dst}/{f}")
        orig = open(f"{REF}/dict_tests/files/{f[:-4]}", "rb").read()
        man["dict"][f] = {"size": len(orig), "sha256": sha(orig), "compressed_size": os.path.getsize(f"{dst}/{f}")}
    # window fixtures: plaintexts are generated in code by the reference tests (tests/mod.rs:582-595)
    dst = os.path.join(HERE, "test_fixtures"); os.makedirs(dst, exist_ok=True)
    fox = b"The quick brown fox jumps over the lazy dog.\n" * 4096
    sphinx = b"Sphinx of black quartz, judge my vow.\n" * 4096
    abc = b"abcdefghijklmnopqrstuvwxyz"
    plain = {"window_128mib.zst": fox, "window_256mib.zst": fox, "window_8mib.zst": sphinx, "abc.txt.zst": abc}
    for f in sorted(os.listdir(f"{REF}/test_fixtures")):
        shutil.copyfile(f"{REF}/test_fixtures/{f}", f"{dst}/{f}")
        p = plain[f]
        man["fixtures"][f] = {"size": len(p), "sha256": sha(p)}
    # fuzz artifacts
    for sub in sorted(os.listdir(f"{REF}/fuzz/artifacts")):
        dst = os.path.join(HERE, "fuzz", sub); os.makedirs(dst, exist_ok=True)
        man["fuzz"][sub] = []
        for f in sorted(os.listdir(f"{REF}/fuzz/artifacts/{sub}")):
            shutil.copyfile(f"{REF}/fuzz/artifacts/{sub}/{f}", f"{dst}/{f}")
            man["fuzz"][sub].append(f)
    json.dump(man, open(os.path.join(HERE, "manifest.json"), "w"), indent=1, sort_keys=True)
    json.dump(chunks, open(os.path.join(HERE, "decodecorpus_originals.json"), "w"), indent=0, sort_keys=True)
    print("corpus", len(man["corpus"]), "dict", len(man["dict"]), "fixtures", len(man["fixtures"]),
          "fuzz", sum(len(v) for v in man["fuzz"].values()))


if __name__ == "__main__":
    main()
