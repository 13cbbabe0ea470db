# TEST INFRASTRUCTURE: the UNMODIFIED field-rate postprocessors as the oracle of ugb200_pp_* (tests/test_field_rate.py).
#   _ref/libfield_rate_ref.so   src/vo_postprocess/temporal-deint.c and interlace.c, each #included where it lies under
#                               $(REF) by a shim of its own (field_rate_*_shim.c) that exposes its static functions,
#                               + src/tv.c, src/utils/{text,random,fs,string}.c; the rest (video_codec.c, video_frame.c, debug.cpp,
#                               tools/ug_stub.c) comes from _ref/libugref.so, built by the Makefile's `ref` target
# Built by __graft_entry__.build() after the Makefile; like it, it needs the reference tree, and _ref/ stays out of git.
REF   ?= /root/reference
CC    := /usr/bin/gcc
OUT   := _ref
CFLAGS_REF := -O3 -msse4.1 -fPIC -D_GNU_SOURCE -I$(REF)/src -fvisibility=default -w -std=gnu2x
FR_C  := src/tv.c src/utils/text.c src/utils/random.c src/utils/fs.c src/utils/string.c

all:
	@if [ -f $(REF)/src/vo_postprocess/temporal-deint.c ] && [ -f $(OUT)/libugref.so ]; then $(MAKE) -f field_rate.mk $(OUT)/libfield_rate_ref.so; \
	 else echo "reference tree absent: using prebuilt $(OUT)/libfield_rate_ref.so if present"; fi

$(OUT)/libfield_rate_ref.so: field_rate_tdeint_shim.c field_rate_interlace_shim.c $(OUT)/libugref.so
	mkdir -p $(OUT)/frobj
	set -e; for f in $(FR_C); do $(CC) $(CFLAGS_REF) -c $(REF)/$$f -o $(OUT)/frobj/$$(echo $$f | tr / _).o; done
	$(CC) $(CFLAGS_REF) -c field_rate_tdeint_shim.c -o $(OUT)/frobj/field_rate_tdeint_shim.o
	$(CC) $(CFLAGS_REF) -c field_rate_interlace_shim.c -o $(OUT)/frobj/field_rate_interlace_shim.o
	$(CC) -shared -o $@ $(OUT)/frobj/*.o -L$(OUT) -lugref -Wl,-rpath,'$$ORIGIN' -Wl,--no-undefined -pthread -lm
