"""Writes tests/golden/run_end_encode.json: the fixed-width and boolean literal cases of arrow-go's
vector_run_end_test.go (TestRunEndFunctions), each for the three run-end types, with the expected run ends and run
values of every chunk.  The expectations are the runs of the reference's literals (the reference builds them with
RunEndEncodedOf + FromJSON); pyarrow.compute.run_end_encode is run over every case as a cross-check.  A null row's
payload is 0 (false), as the reference's builders write it.

    python tests/golden/gen_run_end_encode_golden.py
"""
import json
import os

import pyarrow as pa
import pyarrow.compute as pc

HERE = os.path.dirname(os.path.abspath(__file__))
N, T, F = None, True, False

CASES = [
    # name, value type, chunks, expected [(run_ends, values)] per chunk
    ("simple int32", "int32", [[1, 1, 0, -5, -5, -5, 255, 255]], [([2, 3, 6, 8], [1, 0, -5, 255])]),
    ("uint32 with nulls", "uint32", [[N, 1, 1, N, N, 5]], [([1, 3, 5, 6], [N, 1, N, 5])]),
    ("boolean", "bool", [[T, T, T, F, F]], [([3, 5], [T, F])]),
    ("boolean no runs", "bool", [[T, F, T, F, T, F, T, F, T]], [(list(range(1, 10)), [T, F, T, F, T, F, T, F, T])]),
    ("float64 len=1", "double", [[1.0]], [([1], [1.0])]),
    ("bool chunks", "bool", [[T, T], [T, F, N, N, F], [N, N]], [([2], [T]), ([1, 2, 4, 5], [T, F, N, F]), ([2], [N])]),
    ("float32 chunked", "float", [[1, 1, 0, -5, -5], [-5, 255, 255]], [([2, 3, 5], [1.0, 0.0, -5.0]), ([1, 3], [-5.0, 255.0])]),
    ("empty arrs", "float", [[]], [([], [])]),
    ("empty chunked", "bool", [[], [], []], [([], []), ([], []), ([], [])]),
]
RUN_END_TYPES = ["int16", "int32", "int64"]


def main():
    cases = []
    for name, ty, chunks, expected in CASES:
        for rt in RUN_END_TYPES:
            for chunk, (ends, values) in zip(chunks, expected):
                got = pc.run_end_encode(pa.array(chunk, type=ty), run_end_type=getattr(pa, rt)())
                assert got.run_ends.to_pylist() == ends and got.values.to_pylist() == values, (name, rt, got)
            cases.append({"name": name, "type": ty, "run_end_type": rt, "chunks": chunks,
                          "run_ends": [e for e, _ in expected], "values": [v for _, v in expected]})
    doc = {"_source": "arrow/compute/vector_run_end_test.go:272-286 (TestRunEndFunctions: the fixed-width and boolean cases)",
           "cases": cases}
    with open(os.path.join(HERE, "run_end_encode.json"), "w") as f:
        json.dump(doc, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    main()
