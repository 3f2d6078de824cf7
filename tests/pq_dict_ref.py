"""Python restatement of arrow-go's DictByteArrayEncoder and the column writer's use of it (test oracle only).

  memo table, PutSpaced, dictEncodedSize   parquet/internal/encoding/byte_array_encoder.go:97-135, encoder.go:241-325
  BitWidth, WriteIndices                   encoder.go: 0 for no entries, 1 for one, else bits.Len32(entries - 1)
  checkDictionarySizeLimit                 column_writer_types.gen.go: after every write batch of 1024 slots (batches
                                           restart at every Arrow chunk), DictEncodedSize() >= limit falls back to PLAIN

Every valid value goes through a memo table keyed on its raw bytes, so the entries come in order of first appearance
and the dictionary of any prefix of the slots is a prefix of the whole dictionary.  The dictionary page is the PLAIN
encoding of the entries; a data page's values are its indices at the bit width of the entries when it is flushed.
"""
import numpy as np

import pq_bytearray_ref as B
import pq_encode_model as M

WRITE_BATCH = 1024


def dictionary(vals, valid=None):
    """slot values (bytes) and validity (None: all valid) -> (entries, indices of the valid slots, first-appearance
    flags per slot)"""
    entries, index_of, indices = [], {}, []
    first = np.zeros(len(vals), bool)
    for i, v in enumerate(vals):
        if valid is not None and not valid[i]:
            continue
        v = bytes(v)
        k = index_of.get(v)
        if k is None:
            k = index_of[v] = len(entries)
            entries.append(v)
            first[i] = True
        indices.append(k)
    return entries, np.array(indices, np.uint32), first


def mark_counts(vals, first, marks):
    """[(entries first seen below m, their dictEncodedSize)] for every slot position m"""
    n_before = np.concatenate([[0], np.cumsum(first)])
    size = np.concatenate([[0], np.cumsum([len(v) + 4 if f else 0 for v, f in zip(vals, first)])])
    return [(int(n_before[m]), int(size[m])) for m in marks]


def bit_width(entries):
    return 0 if entries == 0 else 1 if entries == 1 else int(entries - 1).bit_length()


def index_section(indices, entries):
    """the value section of an RLE_DICTIONARY data page: the bit width byte, then the RLE/bit-packed indices"""
    bw = bit_width(entries)
    return bytes([bw]) + M.rle_encode(indices, bw)


def dictionary_page(entries):
    return B.plain_encode(entries)


def batch_ends(chunk_lengths):
    """the slots at which the writer checks the dictionary's size: every 1024 slots of every chunk, and its end"""
    ends, base = [], 0
    for n in chunk_lengths:
        ends += [base + min(k + WRITE_BATCH, n) for k in range(0, n, WRITE_BATCH)]
        base += n
    return ends


def fallback_cut(vals, first, chunk_lengths, limit):
    """the first batch end at which dictEncodedSize >= limit, or None: the dictionary page then holds the entries first
    seen below it, and the slots from it on are written PLAIN"""
    ends = batch_ends(chunk_lengths)
    for e, (_, size) in zip(ends, mark_counts(vals, first, ends)):
        if size >= limit:
            return e
    return None
