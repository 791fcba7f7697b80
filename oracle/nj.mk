# oracle/nj.mk -- the checkers of the -gt nj guide tree.  TEST INFRASTRUCTURE ONLY.
#
#   libnj_oracle.so              nj_oracle.c, our plain-C restatement of NeighborJoining<>::computeTree (always built)
#   _ref/libfamsa_ref_nj.so      ref_nj_harness.cpp, linked against _ref/libfamsa_ref.so (build that first:
#                                make -C oracle all), which holds the UNMODIFIED reference's src/tree/NeighborJoining.cpp.
# The harness is only built where $(REF) exists; the .so travels to the GPU box with the rest of _ref/.
REF      ?= /root/reference
HERE     := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
OUT      := $(HERE)_ref
OBJ      := $(OUT)/obj
CC       ?= gcc
CXX      ?= g++
REFFLAGS := -std=c++20 -O3 -fPIC -pthread -fpermissive -mavx2 -m64 -DARCH_X64 -DSIMD_AVX2 -w \
            -I$(REF)/src -I$(REF)

.PHONY: all
all: $(HERE)libnj_oracle.so $(if $(wildcard $(REF)/src/tree/NeighborJoining.cpp),$(OUT)/libfamsa_ref_nj.so,)

# ISO C, no contraction: every float operation rounded on its own, as in the reference's build
$(HERE)libnj_oracle.so: $(HERE)nj_oracle.c
	$(CC) -O2 -fPIC -shared -std=c11 -ffp-contract=off -Wall -o $@ $<

$(OUT)/libfamsa_ref_nj.so: $(OBJ)/ref_nj_harness.o $(OUT)/libfamsa_ref.so
	$(CXX) -shared -pthread -o $@ $(OBJ)/ref_nj_harness.o -L$(OUT) -lfamsa_ref -Wl,-rpath,'$$ORIGIN'

$(OBJ)/ref_nj_harness.o: $(HERE)ref_nj_harness.cpp
	@mkdir -p $(OBJ)
	$(CXX) $(REFFLAGS) -c $< -o $@
