"""The library's one codec table (ultragrid_b200/csrc/host/video_codec.cpp) against the reference's codec_info[] accessors.

The table is built with g++ and a small extern "C" shim (no CUDA needed) and compared, for every codec id and a set of widths,
with the unmodified video_codec.c in oracle/_ref/libugref.so.
"""
import ctypes
import os
import subprocess

import pytest

import util

HOST = os.path.join(util.ROOT, "ultragrid_b200", "csrc", "host")
SHIM = r'''
#include "video_codec.h"
extern "C" {
int ugb200_pixfmt_supported(int, int) { return 0; }  // get_best_decoder_from's lookup: not under test
int t_count() { return UGB_VIDEO_CODEC_COUNT; }
int t_linesize(unsigned w, int c) { return vc_get_linesize(w, (codec_t) c); }
size_t t_datalen(unsigned w, unsigned h, int c) { return vc_get_datalen(w, h, (codec_t) c); }
int t_block_bytes(int c) { return get_pf_block_bytes((codec_t) c); }
double t_bpp(int c) { return get_bpp((codec_t) c); }
int t_bits(int c) { return get_bits_per_component((codec_t) c); }
bool t_opaque(int c) { return is_codec_opaque((codec_t) c); }
bool t_planar(int c) { return codec_is_planar((codec_t) c); }
const char *t_name(int c) { return get_codec_name((codec_t) c); }
}
'''
WIDTHS = [0, 1, 2, 3, 5, 7, 8, 9, 47, 48, 49, 63, 64, 65, 95, 96, 97, 1919, 1920, 4095, 4096, 7680, (1 << 28) - 1, 1 << 28, (1 << 28) + 1]
HEIGHTS = [1, 2, 1081]
NONE, HW_VDPAU, DRM_PRIME = 0, 23, 41
NO_BYTE_LAYOUT = (HW_VDPAU, DRM_PRIME)  # constant-size handles: every byte size is 0 here


@pytest.fixture(scope="module")
def ours(tmp_path_factory):
    d = tmp_path_factory.mktemp("codec_table")
    src, so = d / "shim.cpp", d / "libcodec_table.so"
    src.write_text(SHIM)
    subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-I", HOST, str(src), os.path.join(HOST, "video_codec.cpp"), "-o", str(so)],
                   check=True, capture_output=True)
    lib = ctypes.CDLL(str(so))
    return _bind(lib, {k: getattr(lib, "t_" + k) for k in TYPES})


@pytest.fixture(scope="module")
def ref():
    path = os.path.join(util.ORACLE_DIR, "_ref", "libugref.so")
    if not os.path.exists(path):
        pytest.skip("oracle/_ref/libugref.so not built (reference tree absent)")
    lib = ctypes.CDLL(path)
    return _bind(lib, {"linesize": lib.vc_get_linesize, "datalen": lib.vc_get_datalen, "block_bytes": lib.get_pf_block_bytes, "bpp": lib.get_bpp,
                       "bits": lib.get_bits_per_component, "opaque": lib.is_codec_opaque, "planar": lib.codec_is_planar, "name": lib.get_codec_name})


_u, _i = ctypes.c_uint, ctypes.c_int
TYPES = {"linesize": ([_u, _i], _i), "datalen": ([_u, _u, _i], ctypes.c_size_t), "block_bytes": ([_i], _i), "bpp": ([_i], ctypes.c_double),
         "bits": ([_i], _i), "opaque": ([_i], ctypes.c_bool), "planar": ([_i], ctypes.c_bool), "name": ([_i], ctypes.c_char_p)}


def _bind(lib, fns):
    for k, (args, res) in TYPES.items():
        fns[k].argtypes, fns[k].restype = args, res
    fns["lib"] = lib
    return fns


def test_table_equals_reference(ours, ref):
    count = ours["lib"].t_count()
    for c in range(count):
        name = ours["name"](c).decode()
        assert name == ref["name"](c).decode(), c
        assert ours["bits"](c) == ref["bits"](c), name
        assert ours["planar"](c) == ref["planar"](c), name
        if c != NONE:  # the reference asserts on is_codec_opaque(NONE)
            assert ours["opaque"](c) == ref["opaque"](c), name
        if c == NONE:  # no block: the reference asserts in get_bpp / get_pf_block_bytes and divides by zero in the sizes
            assert (ours["block_bytes"](c), ours["bpp"](c), ours["linesize"](1920, c), ours["datalen"](1920, 1080, c)) == (0, 0, 0, 0)
            continue
        if c in NO_BYTE_LAYOUT:  # the reference's sizes are the handle's (get_pf_block_bytes asserts where that is 0)
            assert (ours["block_bytes"](c), ours["bpp"](c)) == (0, 0), name
            assert all(ours["linesize"](w, c) == 0 and ours["datalen"](w, 7, c) == 0 for w in WIDTHS), name
            continue
        assert ours["block_bytes"](c) == ref["block_bytes"](c), name
        assert ours["bpp"](c) == ref["bpp"](c), name
        for w in WIDTHS:
            assert ours["linesize"](w, c) == ref["linesize"](w, c), (name, w)
            for h in HEIGHTS:
                got = ours["datalen"](w, h, c)
                if got < 1 << 32:  # the reference multiplies in 32 bits; the table's sizes are 64-bit
                    assert got == ref["datalen"](w, h, c), (name, w, h)


def test_ids_outside_the_table_have_no_layout(ours):
    for c in (-1, ours["lib"].t_count(), 1000):
        assert (ours["linesize"](1920, c), ours["datalen"](1920, 1080, c), ours["block_bytes"](c), ours["bpp"](c), ours["bits"](c)) == (0, 0, 0, 0, 0)
        assert not ours["opaque"](c) and not ours["planar"](c)
        assert ours["name"](c) == b"(unknown)"


def test_sizes_are_64_bit(ours):
    # RG48 at 2^28 pixels is 1.5 GiB a row: a 1080-row frame is past 2^32 bytes, and the filters' frame sizes must not wrap
    assert ours["datalen"](1 << 28, 1080, 27) == 6 * (1 << 28) * 1080
