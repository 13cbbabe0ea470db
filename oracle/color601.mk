# TEST INFRASTRUCTURE: the reference's CPU converters as an UltraGrid run with `--param color-601` sees them, the oracle of
# ugb200_pixfmt_convert_cs(..., UGB_CS_601, ...) (tests/test_color601.py).
#   _ref/libugref601.so   the UNMODIFIED objects of _ref/libugref.so (built by the Makefile's `ref` target from the sources where they lie
#                         under $(REF), with ref_shim.c), linked once more with color601_stub.c in place of the reference's tools/ug_stub.c.
#                         get_commandline_param("color-601") is non-NULL there, so get_color_coeffs(CS_DFL, d) caches and returns BT.601.
# -Bsymbolic binds the objects to the stub and to the `dfl_cs` cache of this library even when libugref.so is loaded in the same process.
# Built by __graft_entry__.build() after the Makefile; it needs the reference tree, and _ref/ stays out of git.
REF   ?= /root/reference
CC    := /usr/bin/gcc
CXX   := /usr/bin/g++
OUT   := _ref
CFLAGS_REF := -O3 -msse4.1 -fPIC -D_GNU_SOURCE -I$(REF)/src -fvisibility=default -w

all:
	@if [ -d $(REF)/src ] && [ -f $(OUT)/libugref.so ]; then $(MAKE) -f color601.mk $(OUT)/libugref601.so; \
	 else echo "reference tree absent: using prebuilt $(OUT)/libugref601.so if present"; fi

$(OUT)/libugref601.so: color601_stub.c $(OUT)/libugref.so
	mkdir -p $(OUT)/obj601
	$(CC) -std=gnu2x $(CFLAGS_REF) -c color601_stub.c -o $(OUT)/obj601/color601_stub.o
	$(CXX) -shared -Wl,-Bsymbolic -o $@ $(filter-out $(OUT)/obj/tools_ug_stub.c.o,$(wildcard $(OUT)/obj/*.o)) $(OUT)/obj601/color601_stub.o -pthread -lm
