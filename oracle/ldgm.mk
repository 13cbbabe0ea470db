# TEST INFRASTRUCTURE: the UNMODIFIED reference LDGM coder as the oracle of include/ugb200_ldgm.h (tests/test_ldgm.py).
#   _ref/libldgm_ref.so   ldgm/src/{ldgm-session,ldgm-session-cpu,tanner}.cpp + ldgm/matrix-gen/{matrix-generator,ldpc-matrix}.cpp, compiled
#                         where they lie under $(REF), + ldgm_ref_shim.cpp (extern "C")
#   _ref/libldgm_fw.so    the module loader and the LDGM_session host side, below
#   _ref/libldgm_gpu_ref.so  the reference GPU coder for sm_90a, below
# Built by __graft_entry__.build() next to the Makefile's targets; like them it needs the reference tree, and _ref/ stays out of git.
REF  ?= /root/reference
CXX  := /usr/bin/g++
OUT  := _ref
LDGM_SRC := ldgm/src/ldgm-session.cpp ldgm/src/ldgm-session-cpu.cpp ldgm/src/tanner.cpp ldgm/matrix-gen/matrix-generator.cpp \
            ldgm/matrix-gen/ldpc-matrix.cpp

all:
	@if [ -d $(REF)/ldgm/src ]; then $(MAKE) -f ldgm.mk $(OUT)/libldgm_ref.so $(OUT)/libldgm_fw.so $(OUT)/libldgm_gpu_ref.so; \
	 else echo "reference tree absent: using prebuilt $(OUT)/libldgm_*.so if present"; fi

$(OUT)/libldgm_ref.so: ldgm_ref_shim.cpp
	mkdir -p $(OUT)
	$(CXX) -O2 -std=gnu++17 -fPIC -shared -w -I$(REF)/ldgm/src -I$(REF)/ldgm/matrix-gen -o $@ ldgm_ref_shim.cpp \
	    $(addprefix $(REF)/,$(LDGM_SRC))

# + ldgm_fw_driver.cpp: the reference's module loader (_ref/libugframework.so, from the Makefile) with the LDGM_session base class and CPU
# coder, into which tests load ultragrid_b200/modules/ultragrid_ldgm_gpu.so
$(OUT)/libldgm_fw.so: ldgm_fw_driver.cpp $(OUT)/libugframework.so
	$(CXX) -O2 -std=gnu++17 -fPIC -shared -w -I$(REF)/src -I$(REF)/ldgm/src -Ifw_stub -o $@ ldgm_fw_driver.cpp \
	    $(addprefix $(REF)/,$(filter ldgm/src/%,$(LDGM_SRC))) -L$(OUT) -lugframework -Wl,-rpath,'$$ORIGIN' -ldl

# the UNMODIFIED reference GPU coder (gpu.cu, ldgm-session-gpu.cpp) with the same nvcc and sm_90a as the product, + ldgm_gpu_ref_shim.cpp
NVCC ?= /usr/local/cuda/bin/nvcc
$(OUT)/libldgm_gpu_ref.so: ldgm_gpu_ref_shim.cpp
	mkdir -p $(OUT)
	$(NVCC) -O3 -gencode arch=compute_90a,code=sm_90a -w -Xcompiler -fPIC -shared -I$(REF)/ldgm/src -o $@ ldgm_gpu_ref_shim.cpp \
	    $(REF)/ldgm/src/gpu.cu $(REF)/ldgm/src/ldgm-session-gpu.cpp $(REF)/ldgm/src/ldgm-session.cpp $(REF)/ldgm/src/tanner.cpp
