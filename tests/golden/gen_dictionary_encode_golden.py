"""Writes tests/golden/dictionary_encode.json: the numeric literal cases of arrow-go's vector_hash_test.go
(TestDictionaryEncode's Mask / Encode index patterns restated on integers, TestDictionaryEncodeChunked, and the
DictEncode cases of the hash kernel tests), each with the expected indices and dictionary, plus one case added here
("encode_chunked": an encoded null that first appears in an earlier chunk than a value), marked "added".  The
expectations of the reference's cases are its literals; pyarrow.compute.dictionary_encode is run over every case as a
cross-check, and is the only check of the added case.

    python tests/golden/gen_dictionary_encode_golden.py
"""
import json
import os

import pyarrow as pa
import pyarrow.compute as pc

HERE = os.path.dirname(os.path.abspath(__file__))

CASES = [
    # name, type, chunks, null_encoding, expected index chunks, expected dictionary
    ("basic", "int64", [[1, 2, 1, 3, 2]], 0, [[0, 1, 0, 2, 1]], [1, 2, 3]),
    ("mod100", "int64", [[i % 100 for i in range(200)]], 0, [[i % 100 for i in range(200)]], list(range(100))),
    ("chunked", "int64", [[1, 2, 1], [2, 3, None]], 0, [[0, 1, 0], [1, 2, None]], [1, 2, 3]),
    ("mask", "int32", [[7, 3, 7, None, 3, None]], 0, [[0, 1, 0, None, 1, None]], [7, 3]),
    ("encode", "int32", [[7, 3, 7, None, 3, None]], 1, [[0, 1, 0, 2, 1, 2]], [7, 3, None]),
    ("encode_chunked", "uint8", [[None, 5], [5, 6, None]], 1, [[0, 1], [1, 2, 0]], [None, 5, 6]),
]
ADDED = {"encode_chunked"}   # not a literal of vector_hash_test.go


def pyarrow_encode(ty, chunks, null_encoding):
    col = pa.chunked_array([pa.array(c, type=ty) for c in chunks], type=ty)
    out = pc.dictionary_encode(col, null_encoding="encode" if null_encoding else "mask")
    dictionary = out.chunk(0).dictionary.to_pylist() if out.num_chunks else []
    return [c.indices.to_pylist() for c in out.chunks], dictionary


def main():
    cases = []
    for name, ty, chunks, ne, indices, dictionary in CASES:
        got_idx, got_dict = pyarrow_encode(ty, chunks, ne)
        assert (got_idx, got_dict) == (indices, dictionary), (name, got_idx, got_dict)
        case = {"name": name, "type": ty, "chunks": chunks, "null_encoding": ne, "indices": indices, "dictionary": dictionary}
        if name in ADDED:
            case["added"] = "not from the reference; expectation cross-checked by pyarrow only"
        cases.append(case)
    doc = {"_source": "arrow/compute/vector_hash_test.go (TestDictionaryEncode, TestDictionaryEncodeChunked, hash kernel DictEncode "
                      "cases), except the cases marked 'added'",
           "cases": cases}
    with open(os.path.join(HERE, "dictionary_encode.json"), "w") as f:
        json.dump(doc, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    main()
