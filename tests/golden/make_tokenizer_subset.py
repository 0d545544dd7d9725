"""Writes tests/golden/tokenizer_subset.json from a llama2.c-format tokenizer.bin (32000 entries).

The tokenizer tests need only part of the 430 KB vocabulary: every entry whose bytes occur in the
texts they encode (so every merge the encoder can consider), the ids they look up directly, the
longest entry, and every string that occurs more than once (first-match lookup).  The tests rebuild
a full-size tokenizer.bin from this subset, with unique placeholders that match no text elsewhere.

  python tests/golden/make_tokenizer_subset.py path/to/tokenizer.bin
"""
import json
import os
import struct
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
VOCAB = 32000
TEXTS = [b"A man dying of thirst is suddenly a mineral water critic?", "中".encode(), "æ".encode()]
IDS = [100, 233]


def main(path):
    with open(path, "rb") as f:
        max_len = struct.unpack("<i", f.read(4))[0]
        entries = []
        for i in range(VOCAB):
            score, n = struct.unpack("<fi", f.read(8))
            entries.append((i, score, f.read(n)))
    count = {}
    for _, _, s in entries:
        count[s] = count.get(s, 0) + 1
    keep = [e for e in entries
            if e[0] in IDS or len(e[2]) == max_len or count[e[2]] > 1 or any(e[2] and e[2] in t for t in TEXTS)]
    with open(os.path.join(HERE, "tokenizer_subset.json"), "w") as f:
        json.dump({"vocab_size": VOCAB, "max_token_len": max_len,
                   "entries": [[i, score, s.hex()] for i, score, s in keep]}, f, separators=(",", ":"))
    print(f"{len(keep)} of {VOCAB} entries kept")


if __name__ == "__main__":
    main(sys.argv[1])
