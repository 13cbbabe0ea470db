"""numpy restatement of UltraGrid's field-rate postprocessors, quirks included.

  double_framerate    src/vo_postprocess/temporal-deint.c:240-277 (perform_df), `:d` through vc_deinterlace_ex
  deinterlace_bob     src/vo_postprocess/temporal-deint.c:279-300 (perform_bob)
  deinterlace_linear  src/vo_postprocess/temporal-deint.c:442-466 (perform_linear) and :307-440 (avg_lines)
  interlace           src/vo_postprocess/interlace.c:159-190 (interlace_postprocess)

`call` 0 is postprocess(in = frame), call 1 the follow-up postprocess(in = NULL); `cur` is the frame just received,
`prev` the one before.  Every function returns a new dst (a copy) with the bytes [0, L) of rows [0, h) that the
reference leaves there; what the reference writes outside them (8/16-bit rows rounded up to 16 bytes, R10k's
4 x L, double_framerate's row h at odd h) is not modelled: it never changes a byte inside them.

contract=False is what the reference computes; contract=True is what ugb200_pp_* compute (include/ugb200.h,
DESIGN.md §8): h < 2 and pitch < L refused (None), opaque codecs refused for linear and `:d`, and `:d` blends with
ugb200_vc_deinterlace_ex's contract (interlace_ref.deinterlace_ex(contract=True)).
"""
import numpy as np

import interlace_ref as IR
from interlace_ref import BITS, R10k, R12L, v210, opaque  # noqa: F401


def _rows(buf, L, h):
    return buf[:L * h].reshape(h, L)


def _put(out, pitch, r, row):
    out[r * pitch:r * pitch + row.size] = row


# ---- row selection: which (source, row) each out row copies; None leaves the row alone -----------------------
def df_rows(h, call):
    """perform_df: call 0 weaves cur's even rows with prev's odd rows (at odd h row h-1 stays unwritten: the even
    loop stops one short while the odd loop writes row h, outside the frame); call 1 is cur"""
    if call == 1:
        return [("cur", r) for r in range(h)]
    return [("prev", r) if r % 2 else (("cur", r) if r + 1 < h else None) for r in range(h)]


def bob_rows(h, call):
    """perform_bob: call 0 doubles rows 0, 2, 4...; call 1 puts row 1 in rows 0-2 and doubles 3, 5...  When a row
    is left over it copies the out row above it (the second copy of the source row two above)."""
    out = []
    for r in range(h):
        rr = h - 2 if r == h - 1 and (h + call) % 2 else r
        out.append(("cur", rr & ~1 if call == 0 else (1 if rr == 0 else (rr - 1) | 1)))
    return out


def interlace_rows(h):
    return [("first", r) if r % 2 == 0 else ("second", r) for r in range(h)]


def _select(srcs, rows, L, h, dst, pitch):
    out = dst.copy()
    for r, sel in enumerate(rows):
        if sel is not None:
            b, s = sel
            _put(out, pitch, r, _rows(srcs[b], L, h)[s])
    return out


# ---- avg_lines ------------------------------------------------------------------------------------------------
def _half_sum(a, b):
    """c1/2 + c2/2 + (c1%2 + c1%2)/2 (:318-319, :334-335): rounds up exactly when the upper sample is odd"""
    return a // 2 + b // 2 + (a & 1)


def avg_lines(codec, a, b):
    """(bytes avg_lines leaves at the start of the out row, their values) for rows a (upper) and b (lower) of L
    bytes; None where it returns false and the caller copies a"""
    L = a.size
    bits = BITS[codec]
    if bits == 8:
        return _half_sum(a.astype(np.uint16), b.astype(np.uint16)).astype(np.uint8)
    if bits == 16:
        assert L % 2 == 0
        return _half_sum(a.view(np.uint16).astype(np.uint32), b.view(np.uint16).astype(np.uint32)).astype(np.uint16).view(np.uint8)
    if codec == v210:  # L/16 groups of 4 words; the bytes after them stay
        n = L // 16 * 16
        x, y = a[:n].view(np.uint32).astype(np.uint64), b[:n].view(np.uint32).astype(np.uint64)
        o = ((x >> 20) + (y >> 20) + 1) // 2 << 20 | ((x >> 10 & 0x3FF) + (y >> 10 & 0x3FF) + 1) // 2 << 10 | \
            ((x & 0x3FF) + (y & 0x3FF) + 1) // 2
        return o.astype(np.uint32).view(np.uint8)
    if codec == R10k:  # words read through ntohl and stored as they come out: byte-swapped, bits 0-1 zero
        assert L % 4 == 0
        x = a.view(np.uint32).byteswap().astype(np.uint64)
        y = b.view(np.uint32).byteswap().astype(np.uint64)
        o = ((x >> 22) + (y >> 22) + 1) // 2 << 22 | ((x >> 12 & 0x3FF) + (y >> 12 & 0x3FF) + 1) // 2 << 12 | \
            ((x >> 2 & 0x3FF) + (y >> 2 & 0x3FF) + 1) // 2 << 2
        return o.astype(np.uint32).view(np.uint8)
    if codec == R12L:
        # L/16 groups of 4 words as one 12-bit little-endian stream; an out word is stored once its last sample is
        # complete, so unless the 4g words end on a sample boundary (g % 3 == 0) the last one is never stored
        g = L // 16
        n = 16 * g if g % 3 == 0 else max(16 * g - 4, 0)
        if n == 0:
            return np.zeros(0, np.uint8)
        span = (n + 2) // 3 * 3
        x = np.zeros(span, np.uint8)
        y = np.zeros(span, np.uint8)
        m = min(span, 16 * g)
        x[:m], y[:m] = a[:m], b[:m]
        return IR._r12l_pack(IR._avg(IR._r12l_unpack(x), IR._r12l_unpack(y)))[:n]
    return None  # DVS10 and the 2- and 4-bit codecs (:436-437)


# ---- the four postprocessors ----------------------------------------------------------------------------------
def _refused(L, h, pitch, contract):
    return contract and (h < 2 or pitch < L)


def double_framerate(codec, prev, cur, L, h, call, dst, pitch, deinterlace=False, contract=False):
    if _refused(L, h, pitch, contract) or (contract and deinterlace and opaque(codec)):
        return None
    out = _select({"prev": prev, "cur": cur}, df_rows(h, call), L, h, dst, pitch)
    if deinterlace:  # vc_deinterlace_ex(out, L, out, L, h) in place, at pitch L whatever the out pitch
        d = IR.deinterlace_ex(codec, out, L, out, L, h, contract)
        if d is None:
            return None if contract else out  # the reference logs and keeps the weave
        out = d
    return out


def bob(cur, L, h, call, dst, pitch, contract=False):
    if _refused(L, h, pitch, contract):
        return None
    return _select({"cur": cur}, bob_rows(h, call), L, h, dst, pitch)


def linear_rows(h, call):
    """perform_linear: ('copy', s) or ('avg', s) (rows s and s+2) for every out row"""
    out = [("copy", 1)] if call == 1 else []
    y = call
    while y < h - 2:
        out += [("copy", y), ("avg", y)]
        y += 2
    while len(out) < h:  # the last row or rows repeat source row y
        out.append(("copy", y))
    return out


def linear(codec, cur, L, h, call, dst, pitch, contract=False):
    if _refused(L, h, pitch, contract) or (contract and opaque(codec)):
        return None
    rows = _rows(cur, L, h)
    out = dst.copy()
    for r, (op, s) in enumerate(linear_rows(h, call)):
        v = avg_lines(codec, rows[s], rows[s + 2]) if op == "avg" else None
        _put(out, pitch, r, rows[s] if v is None else v)
    return out


def interlace(first, second, L, h, dst, pitch, contract=False):
    if _refused(L, h, pitch, contract):
        return None
    return _select({"first": first, "second": second}, interlace_rows(h), L, h, dst, pitch)
