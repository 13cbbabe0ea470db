"""numpy restatement of UltraGrid's linear-blend deinterlacers and field-order converters, quirks included.

  vc_deinterlace_ex   src/video_codec.c:722-854
  vc_deinterlace      src/video_codec.c:597-711 (the SSE2 form an x86-64 build runs)
  il_upper_to_merged  src/video_frame.c:332-355
  il_merged_to_upper  src/video_frame.c:357-379

`deinterlace_ex(..., contract=False)` is what the reference computes; `contract=True` is what
ugb200_vc_deinterlace_ex computes (include/ugb200.h, DESIGN.md §8): 16-bit rows and R12L's whole 36-byte groups
blended in full, opaque codecs refused.
"""
import numpy as np

# codec_t values (src/types.h, include/ugb200.h)
NONE, RGBA, UYVY, YUYV, VUYA, R10k, R12L, v210, DVS10 = range(9)
RGB, BGR, RG48, I420, Y216, Y416 = 12, 20, 27, 29, 30, 31
CODEC_COUNT = 42
# codec_info[] (video_codec.c:120-206): bits per component and VCF_OPAQUE
BITS = [0, 8, 8, 8, 8, 10, 12, 10, 10, 2, 2, 4, 8, 8, 8, 0, 8, 8, 8, 8, 8, 8, 8, 8, 8, 8, 8, 16, 8, 8, 16, 16,
        8, 8, 8, 8, 8, 8, 8, 0, 8, 8]
NON_OPAQUE = (RGBA, UYVY, YUYV, VUYA, R10k, R12L, v210, DVS10, RGB, BGR, RG48, I420, Y216, Y416)


def opaque(codec):
    return codec not in NON_OPAQUE


def _avg(a, b):
    return ((a.astype(np.uint32) + b.astype(np.uint32) + 1) >> 1)


def _r12l_unpack(b):
    """little-endian 12-bit stream: every 3 bytes are 2 samples"""
    t = b.reshape(-1, 3).astype(np.uint32)
    return np.stack([t[:, 0] | (t[:, 1] & 0xF) << 8, t[:, 1] >> 4 | t[:, 2] << 4], axis=1).reshape(-1)


def _r12l_pack(s):
    s = s.reshape(-1, 2)
    out = np.stack([s[:, 0] & 0xFF, (s[:, 0] >> 8) | (s[:, 1] & 0xF) << 4, s[:, 1] >> 4], axis=1)
    return out.astype(np.uint8).reshape(-1)


def _blend_row(codec, src, y, L, contract):
    """(bytes written at the start of out row y, their values) for y < lines - 1"""
    a0 = y * L
    bits = BITS[codec]
    if bits == 8:  # every byte (:745-766)
        return _avg(src[a0:a0 + L], src[a0 + L:a0 + 2 * L]).astype(np.uint8)
    if bits == 16:
        if contract or L < 16:
            # L < 16: the scalar loop over L/2 samples, the second row L/2 samples on (:767-774)
            n, off = L // 2 * 2, (L // 2) * 2
        else:  # only whole 16-byte chunks: the tail loop compares a byte index with a sample count (:755-774)
            n, off = L // 16 * 16, L
        a = src[a0:a0 + n].view(np.uint16)
        b = src[a0 + off:a0 + off + n].view(np.uint16)
        return _avg(a, b).astype(np.uint16).view(np.uint8)
    off = L // 4 * 4  # s32[src_linesize / 4]
    if codec in (v210, R10k):  # whole 16-byte groups of 4 words (:776-823)
        n = L // 16 * 16
        a = src[a0:a0 + n].view(np.uint32).astype(np.uint64)
        b = src[a0 + off:a0 + off + n].view(np.uint32).astype(np.uint64)
        if codec == v210:
            o = ((a >> 20) + (b >> 20) + 1) // 2 << 20 | ((a >> 10 & 0x3FF) + (b >> 10 & 0x3FF) + 1) // 2 << 10 | \
                ((a & 0x3FF) + (b & 0x3FF) + 1) // 2
        else:
            a, b = a.astype(np.uint32).byteswap().astype(np.uint64), b.astype(np.uint32).byteswap().astype(np.uint64)
            o = ((a >> 22) + (b >> 22) + 1) // 2 << 22 | ((a >> 12 & 0x3FF) + (b >> 12 & 0x3FF) + 1) // 2 << 12 | \
                ((a >> 2 & 0x3FF) + (b >> 2 & 0x3FF) + 1) // 2 << 2
            o = o.astype(np.uint32).byteswap()
        return o.astype(np.uint32).view(np.uint8)
    if codec == R12L:
        g = L // 36
        if contract:
            n, off = 36 * g, L
        else:
            # L/36 iterations of 8 words (not 9): a 12-bit stream over the first 32 * g bytes; an output word is
            # stored once its last sample is complete, so the last word waits for a sample that never comes
            # unless 8g words end on a sample boundary (8g % 3 == 0)
            n = 32 * g if g % 3 == 0 else max(32 * g - 4, 0)
        if n == 0:
            return np.zeros(0, np.uint8)
        span = (n + 2) // 3 * 3  # whole sample pairs covering n bytes (the stream reads them)
        a = src[a0:a0 + span]
        b = src[a0 + off:a0 + off + span]
        return _r12l_pack(_avg(_r12l_unpack(a), _r12l_unpack(b)))[:n]
    return None  # DVS10 and every other depth (:849-851)


def deinterlace_ex(codec, src, L, dst, pitch, lines, contract=False):
    """vc_deinterlace_ex: returns the new dst (a copy), or None when refused.  src and dst are flat uint8 arrays;
    for the in-place form pass the same array twice (reads of row y+1 precede its writes in the reference)."""
    if contract and (opaque(codec) or lines == 0 or pitch < L):
        return None
    out = dst.copy()
    if lines == 1:  # :733-736, before any codec check
        out[:L] = src[:L]
        return out
    for y in range(lines - 1):
        r = _blend_row(codec, src, y, L, contract)
        if r is None:
            return None
        out[y * pitch:y * pitch + len(r)] = r
    out[(lines - 1) * pitch:(lines - 1) * pitch + L] = out[(lines - 2) * pitch:(lines - 2) * pitch + L].copy()  # :851
    return out


def _legacy_pass(v, steps):
    if steps == 0:
        return
    a, b = v[0].copy(), v[1].copy()
    for t in range(steps):
        c, d = v[2 * t + 2].copy(), v[2 * t + 3].copy()
        n1 = _avg(_avg(a, c), b).astype(np.uint8)
        v[2 * t + 1] = n1
        n2 = _avg(_avg(n1, d), c).astype(np.uint8)
        v[2 * t + 2] = n2
        a, b = n2, d


def deinterlace(buf, linesize, lines):
    """vc_deinterlace, SSE2 form, linesize >= 16: returns the filtered copy of the linesize * lines bytes"""
    assert linesize >= 16
    v = buf[:linesize * lines].copy().reshape(lines, linesize)
    steps = (lines - 3) // 2 if lines > 4 else 0
    _legacy_pass(v, steps)
    k = 16 - linesize % 16 if linesize % 16 else 0
    if k and steps:
        # the last 16-byte column runs k bytes into the next row, which column 0 has already filtered
        _legacy_pass(v[1:, :k], steps)
    return v.reshape(-1)


def il_upper_to_merged(src, linesize, height):
    v = src[:linesize * height].reshape(height, linesize)
    h = (height + 1) // 2
    out = np.empty_like(v)
    out[0::2], out[1::2] = v[:h], v[h:]
    return out.reshape(-1)


def il_merged_to_upper(src, linesize, height):
    v = src[:linesize * height].reshape(height, linesize)
    h = (height + 1) // 2
    return np.concatenate([v[0::2], v[1::2]]).reshape(-1)
