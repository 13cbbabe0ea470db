# TEST INFRASTRUCTURE: the UNMODIFIED geometry filters as the oracle of ugb200_cf_flip / _mirror / _crop / _split and
# ugb200_pp_border / _interlaced_3d (tests/test_geometry_filters.py).
#   _ref/libgeometry_filters_ref.so   src/capture_filter/{flip.c,mirror.c,split.c}, src/vo_postprocess/{crop.c,split.c,
#                                     border.c,3d-interlaced.c} and src/utils/vf_split.cpp, each #included where it
#                                     lies under $(REF) by a shim of its own (geometry_filters_*_shim.c[pp]) that
#                                     exposes its static functions.  The rest (video_frame.c, video_codec.c,
#                                     pixfmt_conv.c, debug.cpp, color_out.c) comes from _ref/libugref.so, built by the
#                                     Makefile's `ref` target.
# 3d-interlaced.c's inline `pavgb (mem), %xmm0` is legacy SSE, which faults unless the second row is 16-byte
# aligned, so the reference build stops at the first row whenever the line size is not a multiple of 16.  Its shim is
# assembled with -msse2avx: the same instructions VEX-encoded, which compute the same bytes without the alignment
# trap, so the oracle shows what the loop computes at every line size (DESIGN.md §8).
# Built by __graft_entry__.build() after colour_filters.mk; like it, it needs the reference tree, and _ref/ stays out
# of git.
REF   ?= /root/reference
CC    := /usr/bin/gcc
CXX   := /usr/bin/g++
OUT   := _ref
CFLAGS_REF := -O3 -msse4.1 -fPIC -D_GNU_SOURCE -I$(REF)/src -fvisibility=default -w
C_SHIMS := flip mirror crop split vo_split border

all:
	@if [ -f $(REF)/src/vo_postprocess/3d-interlaced.c ] && [ -f $(OUT)/libugref.so ]; then $(MAKE) -f geometry_filters.mk $(OUT)/libgeometry_filters_ref.so; \
	 else echo "reference tree absent: using prebuilt $(OUT)/libgeometry_filters_ref.so if present"; fi

$(OUT)/libgeometry_filters_ref.so: $(foreach s,$(C_SHIMS) 3d,geometry_filters_$(s)_shim.c) geometry_filters_vf_split_shim.cpp $(OUT)/libugref.so
	mkdir -p $(OUT)/geoobj
	set -e; for s in $(C_SHIMS); do $(CC) -std=gnu2x $(CFLAGS_REF) -c geometry_filters_$${s}_shim.c -o $(OUT)/geoobj/$${s}_shim.o; done
	$(CC) -std=gnu2x $(CFLAGS_REF) -Wa,-msse2avx -c geometry_filters_3d_shim.c -o $(OUT)/geoobj/3d_shim.o
	$(CXX) -std=gnu++17 $(CFLAGS_REF) -c geometry_filters_vf_split_shim.cpp -o $(OUT)/geoobj/vf_split_shim.o
	$(CXX) -shared -o $@ $(OUT)/geoobj/*.o -L$(OUT) -lugref -Wl,-rpath,'$$ORIGIN' -Wl,--no-undefined -pthread -lm
