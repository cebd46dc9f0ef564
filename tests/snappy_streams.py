"""A small Snappy writer (google/snappy format_description.txt) that emits every element form on demand, so that tests can hand
the GPU decompressor streams no real compressor would choose: literal lengths in the tag and in 1-4 extra bytes, copies with
1-, 2- and 4-byte offsets, overlapping copies, non-minimal preambles -- and malformed streams, each with the status the device
gives it (csrc/snappy.cuh)."""

BAD_PREAMBLE, LENGTH_MISMATCH, INPUT_OVERRUN, BAD_OFFSET, OUTPUT_OVERRUN, LEFTOVER, SHORT = range(1, 8)


def varint(n, width=None):
    """unsigned LEB128 of n; width pads it with continuation bytes (libsnappy accepts up to 5 bytes)"""
    out = bytearray()
    while True:
        b = n & 0x7F
        n >>= 7
        out.append(b | (0x80 if n else 0))
        if not n:
            break
    while width and len(out) < width:
        out[-1] |= 0x80
        out.append(0)
    return bytes(out)


class Writer:
    """elements appended in order; .output is what a decoder must produce, .stream() the Snappy block"""

    def __init__(self):
        self.elements = bytearray()
        self.output = bytearray()

    def literal(self, data: bytes, extra=None):
        """extra: None puts length - 1 in the tag when it is below 60, else the fewest extra bytes; 1-4 forces that many"""
        n = len(data) - 1
        if extra is None:
            extra = 0 if n < 60 else (1 if n < 1 << 8 else 2 if n < 1 << 16 else 3 if n < 1 << 24 else 4)
        if extra == 0:
            assert n < 60
            self.elements.append(n << 2)
        else:
            self.elements.append((59 + extra) << 2)
            self.elements += n.to_bytes(extra, "little")
        self.elements += data
        self.output += data
        return self

    def copy(self, offset, length, kind=None):
        """kind 1: 1-byte offset (length 4-11, offset < 2048), 2: 2-byte offset, 4: 4-byte offset (length 1-64)"""
        if kind is None:
            kind = 1 if 4 <= length <= 11 and offset < 2048 else (2 if offset < 1 << 16 else 4)
        if kind == 1:
            assert 4 <= length <= 11 and offset < 2048
            self.elements.append(1 | ((length - 4) << 2) | ((offset >> 8) << 5))
            self.elements.append(offset & 0xFF)
        else:
            assert 1 <= length <= 64
            self.elements.append((2 if kind == 2 else 3) | ((length - 1) << 2))
            self.elements += offset.to_bytes(2 if kind == 2 else 4, "little")
        for _ in range(length):                      # byte by byte: an overlapping copy repeats its source
            self.output.append(self.output[len(self.output) - offset] if 0 < offset <= len(self.output) else 0)
        return self

    def raw(self, data: bytes):
        self.elements += data
        return self

    def stream(self, length=None, width=None):
        return varint(len(self.output) if length is None else length, width) + bytes(self.elements)


def valid_streams():
    """name -> (stream, decompressed bytes)"""
    out = {"empty": (b"\x00", b"")}
    lit = bytes(range(256)) * 300
    for n in (1, 2, 59, 60):
        w = Writer().literal(lit[:n])
        out["literal-%d-in-tag" % n] = (w.stream(), bytes(w.output))
    for extra, n in ((1, 61), (1, 256), (2, 257), (2, 65536), (3, 65537), (4, 5), (4, 70000), (3, 1), (2, 1)):
        w = Writer().literal(lit[:n], extra=extra)
        out["literal-%d-with-%d-extra" % (n, extra)] = (w.stream(), bytes(w.output))
    for kind in (1, 2, 4):
        for off in range(1, 9):
            for length in ((4, 7, 11) if kind == 1 else (1, 5, 17, 64)):
                w = Writer().literal(b"abcdefgh"[:off]).copy(off, length, kind)
                out["copy%d-off%d-len%d" % (kind, off, length)] = (w.stream(), bytes(w.output))
    w = Writer().literal(b"0123456789").copy(10, 10, 2).copy(20, 64, 4).copy(84, 11, 1)   # offset == bytes produced so far
    out["offset-equals-produced"] = (w.stream(), bytes(w.output))
    w = Writer().literal(b"x")
    for _ in range(200):
        w.copy(1, 64, 2)                             # a constant run: offset-1 copies, each overlapping the one before
    out["offset-1-run"] = (w.stream(), bytes(w.output))
    w = Writer().literal(b"A").copy(1, 11, 1).literal(b"BC").copy(3, 64, 2).copy(3, 64, 2).copy(7, 9, 1).literal(b"tail")
    out["mixed"] = (w.stream(), bytes(w.output))
    for width in (1, 2, 3, 4, 5):
        w = Writer().literal(b"pre")
        out["preamble-%d-bytes" % width] = (w.stream(width=width), bytes(w.output))
    big = Writer()
    for i in range(3000):                            # more elements than one window of the device's parse
        big.literal(bytes([i & 0xFF, (i >> 8) & 0xFF, 7]))
        big.copy(3 + (i % 5), 4 + (i % 8), 1 if i % 2 else 2)
    out["many-elements"] = (big.stream(), bytes(big.output))
    return out


def malformed_streams():
    """name -> (stream, declared length, status)"""
    ok = Writer().literal(b"abcd")
    return {
        "preamble-truncated": (b"\x80", 0, BAD_PREAMBLE),
        "preamble-overlong-5th-byte": (b"\x80\x80\x80\x80\x10", 0, BAD_PREAMBLE),
        "preamble-6-bytes": (b"\x80\x80\x80\x80\x80\x00", 0, BAD_PREAMBLE),
        "preamble-differs-from-header": (ok.stream(), 5, LENGTH_MISMATCH),
        "literal-past-input": (Writer().raw(b"\x24abc").stream(length=10), 10, INPUT_OVERRUN),
        "literal-length-bytes-cut": (Writer().raw(b"\xf4\x01").stream(length=10), 10, INPUT_OVERRUN),
        "copy-tag-cut": (Writer().literal(b"abcd").raw(b"\x02\x01").stream(length=8), 8, INPUT_OVERRUN),
        "copy-offset-0": (Writer().literal(b"abcd").copy(0, 4, 1).stream(), 8, BAD_OFFSET),
        "copy-before-page-start": (Writer().literal(b"abcd").copy(5, 4, 2).stream(), 8, BAD_OFFSET),
        "output-past-declared": (Writer().literal(b"abcdefgh").stream(length=4), 4, OUTPUT_OVERRUN),
        "copy-past-declared": (Writer().literal(b"abcd").copy(4, 8, 1).stream(length=10), 10, OUTPUT_OVERRUN),
        "bytes-left-over": (Writer().literal(b"abcd").literal(b"e").stream(length=4), 4, LEFTOVER),
        "stream-ends-short": (Writer().literal(b"abcd").stream(length=6), 6, SHORT),
    }
