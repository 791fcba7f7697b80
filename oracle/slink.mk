# oracle/slink.mk -- the reference's -gt slink guide tree for the tests.  TEST INFRASTRUCTURE ONLY.
#
#   _ref/libfamsa_ref_slink.so   ref_slink_harness.cpp, linked against _ref/libfamsa_ref.so (build that first:
#                                make -C oracle all), which holds the UNMODIFIED reference's src/tree/SingleLinkage.cpp.
# Only built where $(REF) exists; the .so travels to the GPU box with the rest of _ref/.
REF      ?= /root/reference
HERE     := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
OUT      := $(HERE)_ref
OBJ      := $(OUT)/obj
CXX      ?= g++
REFFLAGS := -std=c++20 -O3 -fPIC -pthread -fpermissive -mavx2 -m64 -DARCH_X64 -DSIMD_AVX2 -w \
            -I$(REF)/src -I$(REF)

.PHONY: all
all: $(if $(wildcard $(REF)/src/tree/SingleLinkage.cpp),$(OUT)/libfamsa_ref_slink.so,)

$(OUT)/libfamsa_ref_slink.so: $(OBJ)/ref_slink_harness.o $(OUT)/libfamsa_ref.so
	$(CXX) -shared -pthread -o $@ $(OBJ)/ref_slink_harness.o -L$(OUT) -lfamsa_ref -Wl,-rpath,'$$ORIGIN'

$(OBJ)/ref_slink_harness.o: $(HERE)ref_slink_harness.cpp
	@mkdir -p $(OBJ)
	$(CXX) $(REFFLAGS) -c $< -o $@
