# oracle/dist.mk -- the reference's -dist_export path for the tests.  TEST INFRASTRUCTURE ONLY.
#
#   _ref/libfamsa_ref_dist.so   src/tree/DistanceCalculator.cpp of the UNMODIFIED reference under $(REF), compiled
#                               with the flags of oracle/Makefile, plus ref_dist_harness.cpp, linked against
#                               _ref/libfamsa_ref.so (build that first: make -C oracle all).
# Only built where $(REF) exists; the .so travels to the GPU box with the rest of _ref/.
REF      ?= /root/reference
HERE     := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
OUT      := $(HERE)_ref
OBJ      := $(OUT)/obj
CXX      ?= g++
REFFLAGS := -std=c++20 -O3 -fPIC -pthread -fpermissive -mavx2 -m64 -DARCH_X64 -DSIMD_AVX2 -w \
            -I$(REF)/src -I$(REF)

.PHONY: all
all: $(if $(wildcard $(REF)/src/tree/DistanceCalculator.cpp),$(OUT)/libfamsa_ref_dist.so,)

$(OUT)/libfamsa_ref_dist.so: $(OBJ)/tree_DistanceCalculator.o $(OBJ)/ref_dist_harness.o $(OUT)/libfamsa_ref.so
	$(CXX) -shared -pthread -o $@ $(OBJ)/tree_DistanceCalculator.o $(OBJ)/ref_dist_harness.o \
	    -L$(OUT) -lfamsa_ref -Wl,-rpath,'$$ORIGIN'

$(OBJ)/tree_DistanceCalculator.o: $(REF)/src/tree/DistanceCalculator.cpp
	@mkdir -p $(OBJ)
	$(CXX) $(REFFLAGS) -c $< -o $@

$(OBJ)/ref_dist_harness.o: $(HERE)ref_dist_harness.cpp
	@mkdir -p $(OBJ)
	$(CXX) $(REFFLAGS) -c $< -o $@
