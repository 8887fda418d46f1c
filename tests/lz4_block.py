"""A strict LZ4 *block* decoder written from the block format description (lz4_Block_format.md), used to check the
compressor's output.  It rejects offset 0, offsets before the start of the block's output, a block that does not end
with a literals-only sequence, a last match that starts fewer than 12 bytes before the end or ends within the last 5
bytes, and any read past the block's end."""


def _length(blk, i, n):
    """Extends a 4-bit length n (15 = more bytes follow: 255 continues, anything else ends).  Returns (n, i)."""
    if n == 15:
        while True:
            if i >= len(blk):
                raise ValueError("length runs past the end of the block")
            b = blk[i]
            i += 1
            n += b
            if b != 255:
                break
    return n, i


def decode(blk: bytes) -> bytes:
    out = bytearray()
    i = 0
    last_match = None  # (start, end) in the output of the last match
    while True:
        if i >= len(blk):
            raise ValueError("block ends without a literals-only sequence")
        token = blk[i]
        i += 1
        lit, i = _length(blk, i, token >> 4)
        if i + lit > len(blk):
            raise ValueError("literals run past the end of the block")
        out += blk[i:i + lit]
        i += lit
        if i == len(blk):  # the last sequence: literals only
            if token & 15:
                raise ValueError("the last sequence has a match length")
            break
        if i + 2 > len(blk):
            raise ValueError("offset runs past the end of the block")
        off = blk[i] | (blk[i + 1] << 8)
        i += 2
        if off == 0 or off > len(out):
            raise ValueError("offset %d at output position %d" % (off, len(out)))
        mlen, i = _length(blk, i, token & 15)
        mlen += 4
        start = len(out)
        if off >= mlen:
            out += out[start - off:start - off + mlen]
        else:  # an overlapping copy repeats the last `off` bytes
            out += (out[start - off:start] * (mlen // off + 1))[:mlen]
        last_match = (start, len(out))
    if last_match is not None:
        if last_match[0] + 12 > len(out):
            raise ValueError("the last match starts fewer than 12 bytes before the end")
        if last_match[1] + 5 > len(out):
            raise ValueError("the last 5 bytes are not literals")
    return bytes(out)
