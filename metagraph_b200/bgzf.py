"""BGZF member headers read on the host, as mgb_fastx_stage_bgzf's block table reads them (api.cu bgzf_walk): which
files take the device inflate route, and how much text the compressed bytes a reader holds will give."""
import struct

MAX_TEXT = 65536


def block(buf, at=0):
    """The BGZF block at buf[at:]: (compressed size, text size); None when the member there is not a BGZF block;
    "cut" when buf ends inside the member (or before it starts)."""
    h = buf[at:at + 12]
    if len(h) < 12:
        return "cut"
    if h[:4] != b"\x1f\x8b\x08\x04":
        return None
    xlen = struct.unpack_from("<H", h, 10)[0]
    if len(buf) - at < 12 + xlen:
        return "cut"
    p, bsize = 0, None
    while p + 4 <= xlen:
        si, slen = buf[at + 12 + p:at + 14 + p], struct.unpack_from("<H", buf, at + 14 + p)[0]
        if slen > xlen - p - 4:
            break
        if si == b"BC" and slen == 2:
            bsize = struct.unpack_from("<H", buf, at + 16 + p)[0]
        p += 4 + slen
    if p != xlen or bsize is None or bsize + 1 < 12 + xlen + 8:
        return None
    size = bsize + 1
    if len(buf) - at < size:
        return "cut"
    isize = struct.unpack_from("<I", buf, at + size - 4)[0]
    return (size, isize) if isize <= MAX_TEXT else None


def text_of(buf, limit=None):
    """(text of the complete BGZF blocks at the start of buf, up to `limit`; whether a member that is not one follows)"""
    at = text = 0
    while limit is None or text < limit:
        b = block(buf, at)
        if b == "cut":
            return text, False
        if b is None:
            return text, True
        at += b[0]
        text += b[1]
    return text, False


def is_bgzf(path):
    """whether the file's first member is a complete BGZF block"""
    with open(path, "rb") as f:
        head = f.read(65536 + 8)
    b = block(head)
    return b is not None and b != "cut"
