# TEST INFRASTRUCTURE: the UNMODIFIED colour capture filters as the oracle of ugb200_cf_* (tests/test_colour_filters.py).
#   _ref/libcolour_filters_ref.so   src/capture_filter/{gamma.cpp,matrix.c,matrix2.c,grayscale.c}, each #included where
#                                   it lies under $(REF) by a shim of its own (colour_filters_*_shim.c[pp]) that exposes
#                                   its static functions; gamma.cpp is built with g++.  The rest (worker.cpp,
#                                   video_frame.c, pixfmt_conv.c, debug.cpp, color_out.c) comes from _ref/libugref.so,
#                                   built by the Makefile's `ref` target.
# Built by __graft_entry__.build() after field_rate.mk; like it, it needs the reference tree, and _ref/ stays out of git.
REF   ?= /root/reference
CC    := /usr/bin/gcc
CXX   := /usr/bin/g++
OUT   := _ref
CFLAGS_REF := -O3 -msse4.1 -fPIC -D_GNU_SOURCE -I$(REF)/src -fvisibility=default -w
SHIMS := colour_filters_matrix_shim.c colour_filters_matrix2_shim.c colour_filters_grayscale_shim.c colour_filters_gamma_shim.cpp

all:
	@if [ -f $(REF)/src/capture_filter/matrix2.c ] && [ -f $(OUT)/libugref.so ]; then $(MAKE) -f colour_filters.mk $(OUT)/libcolour_filters_ref.so; \
	 else echo "reference tree absent: using prebuilt $(OUT)/libcolour_filters_ref.so if present"; fi

$(OUT)/libcolour_filters_ref.so: $(SHIMS) $(OUT)/libugref.so
	mkdir -p $(OUT)/cfobj
	$(CC) -std=gnu2x $(CFLAGS_REF) -c colour_filters_matrix_shim.c -o $(OUT)/cfobj/matrix_shim.o
	$(CC) -std=gnu2x $(CFLAGS_REF) -c colour_filters_matrix2_shim.c -o $(OUT)/cfobj/matrix2_shim.o
	$(CC) -std=gnu2x $(CFLAGS_REF) -c colour_filters_grayscale_shim.c -o $(OUT)/cfobj/grayscale_shim.o
	$(CXX) -std=gnu++17 $(CFLAGS_REF) -c colour_filters_gamma_shim.cpp -o $(OUT)/cfobj/gamma_shim.o
	$(CXX) -shared -o $@ $(OUT)/cfobj/*.o -L$(OUT) -lugref -Wl,-rpath,'$$ORIGIN' -Wl,--no-undefined -pthread -lm
