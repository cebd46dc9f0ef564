"""CPU ORACLE (test infrastructure): the Parquet BYTE_ARRAY and DELTA_* page decoding, restated from the reference's vectorized
readers (SQLJ = sql/core/src/main/java/org/apache/spark/sql/execution/datasources/parquet).  It extends oracle/parquet_oracle.py
(the RLE / bit-packed hybrid, PLAIN and dictionary pages of fixed-width columns), whose helpers it reuses, and is pinned in
tests/test_scan_strings_cpu.py against files written and read back by pyarrow (parquet-cpp) and one written by parquet-mr.

Encodings are the SB_ENC_* numbers of the page descriptors (include/spark_b200.h)."""
import numpy as np

from oracle import parquet_oracle as PO

BYTE_ARRAY = 6
ENC_PLAIN, ENC_RLE_DICTIONARY, ENC_RLE_BOOLEAN, ENC_DELTA_BINARY_PACKED, ENC_DELTA_LENGTH_BYTE_ARRAY, ENC_DELTA_BYTE_ARRAY = range(6)
_M64 = (1 << 64) - 1


def _zigzag(z):
    return (z >> 1) ^ -(z & 1)


def decode_delta_binary_packed(buf, pos=0):
    """DELTA_BINARY_PACKED stream at buf[pos:] -> (values as Python ints wrapped to signed 64 bits, position after the stream).
    SQLJ/VectorizedDeltaBinaryPackedReader.java:
      :91-122 initFromPage -- <block size in values> <miniblocks per block> <total value count> as unsigned varints, then the
              first value as a zig-zag varint; miniblock size = block size / miniblocks;
      :457-467 readBlockHeader -- the block's zig-zag min delta, then (:492-500 readBitWidthsForMiniBlocks) one bit-width byte for
              EVERY miniblock of the block, the last block's unused ones included;
      :474-489 unpackMiniBlock -- a whole miniblock of LSB-first packed values, read only when one of its values is needed (so
              the bodies of the last block's unused miniblocks are not in the stream);
      :428-454 loadMiniBlockToOutput -- value = previous value + min delta + packed value, in long arithmetic (wrapping)."""
    b = np.asarray(buf, dtype=np.uint8)
    block, pos = PO.read_uvarint(b, pos)
    minis, pos = PO.read_uvarint(b, pos)
    total, pos = PO.read_uvarint(b, pos)
    z, pos = PO.read_uvarint(b, pos)
    vpm = block // minis
    out = [_zigzag(z) & _M64] if total > 0 else []
    while len(out) < total:
        z, pos = PO.read_uvarint(b, pos)
        min_delta = _zigzag(z)
        widths = [int(x) for x in b[pos:pos + minis]]
        pos += minis
        for bw in widths:
            if len(out) >= total:
                break
            nbytes = vpm * bw // 8
            bits = np.unpackbits(b[pos:pos + nbytes], bitorder="little").astype(object)
            pos += nbytes
            weights = [1 << k for k in range(bw)]
            for j in range(vpm):
                if len(out) >= total:
                    break
                packed = sum(int(x) * w for x, w in zip(bits[j * bw:(j + 1) * bw], weights))
                out.append((out[-1] + min_delta + packed) & _M64)
    return [v - (1 << 64) if v >> 63 else v for v in out], pos


def decode_plain_byte_arrays(buf, count, pos=0):
    """PLAIN BYTE_ARRAY values (SQLJ/VectorizedPlainValuesReader.java:519-531 readBinary: a 4-byte little-endian length, then
    the bytes) -> (list of bytes, position after them)."""
    b = bytes(np.asarray(buf, dtype=np.uint8))
    out = []
    for _ in range(count):
        n = int.from_bytes(b[pos:pos + 4], "little")
        out.append(b[pos + 4:pos + 4 + n])
        pos += 4 + n
    return out, pos


def decode_delta_length_byte_array(buf, pos=0):
    """SQLJ/VectorizedDeltaLengthByteArrayReader.java:48-53 initFromPage: DELTA_BINARY_PACKED lengths, then the values' bytes
    concatenated -> (list of bytes, position after them)."""
    lens, pos = decode_delta_binary_packed(buf, pos)
    b = bytes(np.asarray(buf, dtype=np.uint8))
    out = []
    for n in lens:
        out.append(b[pos:pos + n])
        pos += n
    return out, pos


def decode_delta_byte_array(buf):
    """SQLJ/VectorizedDeltaByteArrayReader.java: :60-66 initFromPage -- prefix lengths as DELTA_BINARY_PACKED, then the suffixes
    as DELTA_LENGTH_BYTE_ARRAY; :74-98 readValues -- value i = the first prefix[i] bytes of value i-1, then its suffix."""
    prefix, pos = decode_delta_binary_packed(buf, 0)
    suffix, _ = decode_delta_length_byte_array(buf, pos)
    out, prev = [], b""
    for p, s in zip(prefix, suffix):
        prev = prev[:p] + s
        out.append(prev)
    return out


def decode_byte_array_chunk(data, pages, dict_offset, dict_count):
    """A BYTE_ARRAY column chunk -> one `bytes` per row, None at NULL rows.  Dictionary pages hold PLAIN byte arrays
    (SQLJ/VectorizedRleValuesReader.java:834, the dictionary ids of a binary column)."""
    data = np.asarray(data, dtype=np.uint8)
    dictionary = decode_plain_byte_arrays(data, dict_count, dict_offset)[0] if dict_offset >= 0 else None
    rows = []
    for enc, n, voff, vbytes, doff, dbytes in pages:
        valid = PO.decode_hybrid(data[doff:doff + dbytes], 1, n).astype(bool) if dbytes > 0 else np.ones(n, bool)
        nvals = int(valid.sum())
        body = data[voff:voff + vbytes]
        if nvals == 0:
            dense = []
        elif enc == ENC_PLAIN:
            dense = decode_plain_byte_arrays(body, nvals)[0]
        elif enc == ENC_RLE_DICTIONARY:
            dense = [dictionary[i] for i in PO.decode_hybrid(body[1:], int(body[0]), nvals)]
        elif enc == ENC_DELTA_LENGTH_BYTE_ARRAY:
            dense = decode_delta_length_byte_array(body)[0]
        elif enc == ENC_DELTA_BYTE_ARRAY:
            dense = decode_delta_byte_array(body)
        else:
            raise ValueError("encoding %d is not a BYTE_ARRAY encoding" % enc)
        it = iter(dense)
        rows.extend(next(it) if v else None for v in valid)
    return rows


def decode_column_chunk(data, pages, dict_offset, dict_count, physical):
    """oracle.parquet_oracle.decode_column_chunk, extended: physical BYTE_ARRAY -> (list of bytes / None, None); INT32 / INT64
    pages in DELTA_BINARY_PACKED (INT32 keeps the low 32 bits of the 64-bit running sum) are decoded here, the other pages
    there."""
    if physical == BYTE_ARRAY:
        return decode_byte_array_chunk(data, pages, dict_offset, dict_count), None
    if not any(p[0] == ENC_DELTA_BINARY_PACKED for p in pages):
        return PO.decode_column_chunk(data, pages, dict_offset, dict_count, physical)
    data = np.asarray(data, dtype=np.uint8)
    dt = np.dtype("<i4") if physical == 1 else np.dtype("<i8")
    vals, valids, nullable = [], [], False
    for page in pages:
        enc, n, voff, vbytes, doff, dbytes = page
        if enc != ENC_DELTA_BINARY_PACKED:
            v, ok = PO.decode_column_chunk(data, [page], dict_offset, dict_count, physical)
            vals.append(v.astype(dt))
            valids.append(ok if ok is not None else np.ones(n, bool))
            nullable |= ok is not None
            continue
        valid = PO.decode_hybrid(data[doff:doff + dbytes], 1, n).astype(bool) if dbytes > 0 else np.ones(n, bool)
        nullable |= dbytes > 0
        dense = np.array(decode_delta_binary_packed(data[voff:voff + vbytes])[0][: int(valid.sum())], dtype=object)
        dense = np.array([int(x) & 0xFFFFFFFF for x in dense], dtype=np.uint64).astype(np.uint32).view(np.int32) if dt.itemsize == 4 \
            else np.array(list(dense), dtype=np.int64)
        row = np.zeros(n, dt)
        row[valid] = dense
        vals.append(row)
        valids.append(valid)
    return np.concatenate(vals), (np.concatenate(valids) if nullable else None)
