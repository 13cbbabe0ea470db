# TEST INFRASTRUCTURE: the UNMODIFIED logo and R12L <-> Y416 pass-through filters as the oracle of ugb200_cf_logo,
# ugb200_cf_r12l_to_y416_fake and ugb200_pp_y416_to_r12l_fake (tests/test_logo_filters.py).
#   _ref/liblogo_filters_ref.so   src/capture_filter/{logo.c,r12l_to_y416_fake.c} and
#                                 src/vo_postprocess/y416_to_r12l_fake.c, each #included where it lies under $(REF) by
#                                 a shim of its own (logo_filters_*_shim.c) that exposes its static functions.  The
#                                 rest (pam.c, pixfmt_conv.c, video_frame.c, video_codec.c, worker.cpp, misc.cpp,
#                                 debug.cpp, color_out.c) comes from _ref/libugref.so, built by the Makefile's `ref`
#                                 target.
# Built by __graft_entry__.build() after geometry_filters.mk; like it, it needs the reference tree, and _ref/ stays
# out of git.
REF   ?= /root/reference
CC    := /usr/bin/gcc
CXX   := /usr/bin/g++
OUT   := _ref
CFLAGS_REF := -O3 -msse4.1 -fPIC -D_GNU_SOURCE -I$(REF)/src -fvisibility=default -w
SHIMS := logo r12l y416

all:
	@if [ -f $(REF)/src/vo_postprocess/y416_to_r12l_fake.c ] && [ -f $(OUT)/libugref.so ]; then $(MAKE) -f logo_filters.mk $(OUT)/liblogo_filters_ref.so; \
	 else echo "reference tree absent: using prebuilt $(OUT)/liblogo_filters_ref.so if present"; fi

$(OUT)/liblogo_filters_ref.so: $(foreach s,$(SHIMS),logo_filters_$(s)_shim.c) $(OUT)/libugref.so
	mkdir -p $(OUT)/logoobj
	set -e; for s in $(SHIMS); do $(CC) -std=gnu2x $(CFLAGS_REF) -c logo_filters_$${s}_shim.c -o $(OUT)/logoobj/$${s}_shim.o; done
	$(CXX) -shared -o $@ $(OUT)/logoobj/*.o -L$(OUT) -lugref -Wl,-rpath,'$$ORIGIN' -Wl,--no-undefined -pthread -lm
