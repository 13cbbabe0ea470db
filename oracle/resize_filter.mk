# TEST INFRASTRUCTURE: the UNMODIFIED resize filter as the oracle of everything ugb200_cf_resize takes from resize.c
# (tests/test_resize_filter.py): option parsing, the decode route, the output descriptor and the bytes handed to the
# resampler.
#   _ref/libresize_filter_ref.so   src/capture_filter/resize.c, #included where it lies under $(REF) by
#                                  resize_filter_shim.c, which stands in for resize_utils.cpp (OpenCV): its
#                                  resize_frame records what it is handed, its resize_algo_from_string parses the five
#                                  names and `help`.  The rest (video_codec.c, video_frame.c, pixfmt_conv.c,
#                                  parallel_conv.c, color_out.c, debug.cpp ...) comes from _ref/libugref.so, built by the
#                                  Makefile's `ref` target.
# Built by __graft_entry__.build() after logo_filters.mk; like it, it needs the reference tree, and _ref/ stays out of git.
REF   ?= /root/reference
CC    := /usr/bin/gcc
CXX   := /usr/bin/g++
OUT   := _ref
CFLAGS_REF := -O3 -msse4.1 -fPIC -D_GNU_SOURCE -I$(REF)/src -fvisibility=default -w

all:
	@if [ -f $(REF)/src/capture_filter/resize.c ] && [ -f $(OUT)/libugref.so ]; then $(MAKE) -f resize_filter.mk $(OUT)/libresize_filter_ref.so; \
	 else echo "reference tree absent: using prebuilt $(OUT)/libresize_filter_ref.so if present"; fi

$(OUT)/libresize_filter_ref.so: resize_filter_shim.c $(OUT)/libugref.so
	mkdir -p $(OUT)/resizeobj
	$(CC) -std=gnu2x $(CFLAGS_REF) -c resize_filter_shim.c -o $(OUT)/resizeobj/resize_filter_shim.o
	$(CXX) -shared -o $@ $(OUT)/resizeobj/resize_filter_shim.o -L$(OUT) -lugref -Wl,-rpath,'$$ORIGIN' -Wl,--no-undefined -pthread -lm
