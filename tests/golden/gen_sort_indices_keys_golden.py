"""Writes tests/golden/sort_indices_keys.json: the reference's literal sort_indices vectors whose key columns are
numeric or boolean (arrow/compute/vector_sort_test.go:554-1665); LEFT_OUT names every other case of that range and
why it is not here.  Columns the keys do not use are dropped, so column indices count the kept columns.  A column is a list of chunks; a value is a number, "NaN" or null (a null row).
Keys are [column, order (0 asc, 1 desc), null placement (0 at end, 1 at start)].  kind is the reference's input:
"array" and "chunked" (one column, the first key), "record" or "table".

    python tests/golden/gen_sort_indices_keys_golden.py
"""
import json
import os

NAN = "NaN"
AB_END = [[0, 0, 0], [1, 1, 0]]      # cppRecordKeysAB(NullsAtEnd)
AB_START = [[0, 0, 1], [1, 1, 1]]    # cppRecordKeysAB(NullsAtStart)
NULL_A = [None, 1, 3, None, 2, 1, 3]
NULL_B = [5, 3, None, None, 5, 5, 5]
NN_A = [None, 1, 3, None, NAN, NAN, NAN, 1]
NN_B = [5, 3, None, None, None, NAN, 5, 5]
DUP = [[0, 0, 0], [1, 1, 0], [0, 0, 0], [1, 0, 0], [0, 1, 0]]
I16 = [0, 1, None, -3, None, -42, 5]
F64 = [None, 1, 3.3, None, 2, 5.3]
U8 = [255, None, 0, 255, 10, None, 128, 0]
U8_CHUNKS = [[None, 1], [3, None, 2], [1]]


def case(name, kind, types, columns, keys, want):
    return {"name": name, "kind": kind, "types": types, "columns": columns, "keys": keys, "want": want}


CASES = [
    case("TestSortRecordBatch/SortBySecondColumn", "record", ["int32", "int32"],
         [[[30, 10, 20]], [[1, 2, 3]]], [[0, 0, 0]], [1, 2, 0]),
    case("TestSortRecordBatch/MultiColumnLexicographic", "record", ["int32", "int32"],
         [[[1, 1, 2, 2]], [[100, 200, 300, 400]]], [[0, 0, 0], [1, 1, 1]], [1, 0, 3, 2]),
    case("TestSortTable/SortBySecondColumn", "table", ["int32"], [[[30, 25, 35]]], [[0, 0, 0]], [1, 0, 2]),
    case("TestSortTable/MultiColumnSort", "table", ["int32", "int32"],
         [[[2, 1, 1, 2]], [[100, 200, 300, 400]]], [[0, 0, 0], [1, 1, 1]], [2, 1, 3, 0]),
    case("TestSortIndicesChunked/Int32ChunkedAscending", "chunked", ["int32"], [[[3, 1], [4, 1, 5]]], [[0, 0, 0]],
         [1, 3, 0, 2, 4]),
    case("TestSortIndicesChunked/Float64ChunkedWithNaN", "chunked", ["float64"], [[[1.0, NAN], [2.0, 0.5]]], [[0, 0, 0]],
         [3, 0, 2, 1]),
    case("TestVectorSortIndicesCppArrayParity/Int16NullsDefaultAndDescendingAtStart/AscAtEnd", "array", ["int16"],
         [[I16]], [[0, 0, 0]], [5, 3, 0, 1, 6, 2, 4]),
    case("TestVectorSortIndicesCppArrayParity/Int16NullsDefaultAndDescendingAtStart/DescAtStart", "array", ["int16"],
         [[I16]], [[0, 1, 1]], [2, 4, 6, 1, 0, 3, 5]),
    case("TestVectorSortIndicesCppArrayParity/Float64NullNaNMatchesCppRealSuite/AscAtEnd", "array", ["float64"],
         [[F64]], [[0, 0, 0]], [1, 4, 2, 5, 0, 3]),
    case("TestVectorSortIndicesCppArrayParity/Float64NullNaNMatchesCppRealSuite/AscAtStart", "array", ["float64"],
         [[F64]], [[0, 0, 1]], [0, 3, 1, 4, 2, 5]),
    case("TestVectorSortIndicesCppArrayParity/Float64NullNaNMatchesCppRealSuite/DescAtEnd", "array", ["float64"],
         [[F64]], [[0, 1, 0]], [5, 2, 4, 1, 0, 3]),
    case("TestVectorSortIndicesCppArrayParity/Float64NullNaNMatchesCppRealSuite/DescAtStart", "array", ["float64"],
         [[F64]], [[0, 1, 1]], [0, 3, 5, 2, 4, 1]),
    case("TestVectorSortIndicesCppArrayParity/UInt8TieBreakSmallRange/AscAtEnd", "array", ["uint8"],
         [[U8]], [[0, 0, 0]], [2, 7, 4, 6, 0, 3, 1, 5]),
    case("TestVectorSortIndicesCppArrayParity/UInt8TieBreakSmallRange/AscAtStart", "array", ["uint8"],
         [[U8]], [[0, 0, 1]], [1, 5, 2, 7, 4, 6, 0, 3]),
    case("TestVectorSortIndicesCppChunkedParity/Int16ContiguousEqualsSingleArray/AscAtEnd", "chunked", ["int16"],
         [[I16[:2], I16[2:]]], [[0, 0, 0]], [5, 3, 0, 1, 6, 2, 4]),
    case("TestVectorSortIndicesCppChunkedParity/Int16ContiguousEqualsSingleArray/DescAtStart", "chunked", ["int16"],
         [[I16[:2], I16[2:]]], [[0, 1, 1]], [2, 4, 6, 1, 0, 3, 5]),
    case("TestVectorSortIndicesCppChunkedParity/Uint8NullsAcrossChunks/AscAtEnd", "chunked", ["uint8"],
         [U8_CHUNKS], [[0, 0, 0]], [1, 5, 4, 2, 0, 3]),
    case("TestVectorSortIndicesCppChunkedParity/Uint8NullsAcrossChunks/AscAtStart", "chunked", ["uint8"],
         [U8_CHUNKS], [[0, 0, 1]], [0, 3, 1, 5, 4, 2]),
    case("TestVectorSortIndicesCppChunkedParity/Uint8NullsAcrossChunks/DescAtEnd", "chunked", ["uint8"],
         [U8_CHUNKS], [[0, 1, 0]], [2, 4, 1, 5, 0, 3]),
    case("TestVectorSortIndicesCppChunkedParity/Uint8NullsAcrossChunks/DescAtStart", "chunked", ["uint8"],
         [U8_CHUNKS], [[0, 1, 1]], [0, 3, 2, 4, 1, 5]),
    case("TestSortTableChunked/MisalignedChunksMultiColumnLexicographic", "table", ["int32", "int32"],
         [[[10, 20], [15]], [[1, 2, 3]]], [[0, 0, 0], [1, 0, 0]], [0, 2, 1]),
    case("TestVectorSortIndicesCppRecordBatchParity/NoNull/AtEnd", "record", ["uint8", "uint32"],
         [[[3, 1, 3, 0, 2, 1, 1]], [[5, 3, 4, 6, 5, 5, 3]]], AB_END, [3, 5, 1, 6, 4, 0, 2]),
    case("TestVectorSortIndicesCppRecordBatchParity/NoNull/AtStart", "record", ["uint8", "uint32"],
         [[[3, 1, 3, 0, 2, 1, 1]], [[5, 3, 4, 6, 5, 5, 3]]], AB_START, [3, 5, 1, 6, 4, 0, 2]),
    case("TestVectorSortIndicesCppRecordBatchParity/Null/AtEnd", "record", ["uint8", "uint32"],
         [[NULL_A], [NULL_B]], AB_END, [5, 1, 4, 6, 2, 0, 3]),
    case("TestVectorSortIndicesCppRecordBatchParity/Null/AtStart", "record", ["uint8", "uint32"],
         [[NULL_A], [NULL_B]], AB_START, [3, 0, 5, 1, 4, 2, 6]),
    case("TestVectorSortIndicesCppRecordBatchParity/NaN/AtEnd", "record", ["float32", "float64"],
         [[[3, 1, 3, 0, NAN, NAN, NAN, 1]], [[5, NAN, 4, 6, 5, NAN, 5, 5]]], AB_END, [3, 7, 1, 0, 2, 4, 6, 5]),
    case("TestVectorSortIndicesCppRecordBatchParity/NaN/AtStart", "record", ["float32", "float64"],
         [[[3, 1, 3, 0, NAN, NAN, NAN, 1]], [[5, NAN, 4, 6, 5, NAN, 5, 5]]], AB_START, [5, 4, 6, 3, 1, 7, 0, 2]),
    case("TestVectorSortIndicesCppRecordBatchParity/NaNAndNull/AtEnd", "record", ["float32", "float64"],
         [[NN_A], [NN_B]], AB_END, [7, 1, 2, 6, 5, 4, 0, 3]),
    case("TestVectorSortIndicesCppRecordBatchParity/NaNAndNull/AtStart", "record", ["float32", "float64"],
         [[NN_A], [NN_B]], AB_START, [3, 0, 4, 5, 6, 7, 1, 2]),
    case("TestVectorSortIndicesCppRecordBatchParity/Boolean/AtEnd", "record", ["bool", "bool"],
         [[[True, False, True, False, True, None, False, None]], [[None, None, True, True, False, False, None, True]]],
         AB_END, [3, 1, 6, 2, 4, 0, 7, 5]),
    case("TestVectorSortIndicesCppRecordBatchParity/Boolean/AtStart", "record", ["bool", "bool"],
         [[[True, False, True, False, True, None, False, None]], [[None, None, True, True, False, False, None, True]]],
         AB_START, [7, 5, 1, 6, 3, 0, 2, 4]),
    case("TestVectorSortIndicesCppRecordBatchParity/DuplicateSortKeys/AtEnd", "record", ["float32", "float64"],
         [[NN_A], [NN_B]], DUP, [7, 1, 2, 6, 5, 4, 0, 3]),
    case("TestVectorSortIndicesCppRecordBatchParity/DuplicateSortKeys/AtStart", "record", ["float32", "float64"],
         [[NN_A], [NN_B]], [[c, o, 1] for c, o, _ in DUP], [3, 0, 4, 5, 6, 7, 1, 2]),
    case("TestVectorSortIndicesCppTableParity/EmptyTable", "table", ["uint8", "uint32"],
         [[[]], [[]]], AB_END, []),
    case("TestVectorSortIndicesCppTableParity/NullSingleAndMultiChunk/AtEnd", "table", ["uint8", "uint32"],
         [[NULL_A[:3], NULL_A[3:]], [NULL_B[:3], NULL_B[3:]]], AB_END, [5, 1, 4, 6, 2, 0, 3]),
    case("TestVectorSortIndicesCppTableParity/NullSingleAndMultiChunk/AtStart", "table", ["uint8", "uint32"],
         [[NULL_A[:3], NULL_A[3:]], [NULL_B[:3], NULL_B[3:]]], AB_START, [3, 0, 5, 1, 4, 2, 6]),
]

LEFT_OUT = {
    "TestVectorSortIndicesCppRecordBatchParity/MoreTypes": "timestamp, large_string and fixed_size_binary keys",
    "TestVectorSortIndicesCppRecordBatchParity/Decimal": "decimal128 / decimal256 keys",
    "TestVectorSortIndicesCppTableParity/BinaryLikeTwoChunks": "binary-like keys",
    "TestSortIndicesChunked/StringChunkedWithNulls": "string key",
    "TestSortTableChunked/MultiChunkSingleColumn": "string key",
    "TestSortTableChunked/MultiChunkMultiColumn": "string key (the second of its three keys)",
    "TestVectorSortIndicesCppArrayParity/FixedSizeBinaryMatchesCpp": "fixed_size_binary key",
    "TestSortRecordBatch/InvalidColumnIndex": "an error case, covered by the error tests",
    "TestVectorSortIndicesCppTableParity/EmptySortKeysInvalid": "an error case, covered by the error tests",
    "TestVectorSortIndicesCppChunkedParity/Float32NaNAcrossChunks": "skipped by the reference itself (NaN order of chunk merges)",
}

if __name__ == "__main__":
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "sort_indices_keys.json")
    with open(path, "w") as f:
        json.dump({"source": "arrow/compute/vector_sort_test.go", "cases": CASES, "left_out": LEFT_OUT}, f, indent=1)
        f.write("\n")
