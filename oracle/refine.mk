# oracle/refine.mk -- the reference's refinement (CFAMSA::RefineAlignment + CalculateTotalScore) for the tests.  TEST INFRASTRUCTURE ONLY.
#
#   _ref/libfamsa_ref_refine.so   ref_refine_harness.cpp, linked against _ref/libfamsa_ref.so (build that first:
#                                make -C oracle all), which holds the UNMODIFIED reference's CProfile.
# Only built where $(REF) exists; the .so travels to the GPU box with the rest of _ref/.
REF      ?= /root/reference
HERE     := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
OUT      := $(HERE)_ref
OBJ      := $(OUT)/obj
CXX      ?= g++
REFFLAGS := -std=c++20 -O3 -fPIC -pthread -fpermissive -mavx2 -m64 -DARCH_X64 -DSIMD_AVX2 -w \
            -I$(REF)/src -I$(REF)

# The object is named by a checksum of the harness source, so a _ref/ carried over from a build of another revision is
# rebuilt whatever the files' modification times say.
HSUM     := $(firstword $(shell cksum < $(HERE)ref_refine_harness.cpp))
HOBJ     := $(OBJ)/ref_refine_harness-$(HSUM).o

.PHONY: all
all: $(if $(wildcard $(REF)/src/core/profile.cpp),$(OUT)/libfamsa_ref_refine.so,)

$(OUT)/libfamsa_ref_refine.so: $(HOBJ) $(OUT)/libfamsa_ref.so
	$(CXX) -shared -pthread -o $@ $(HOBJ) -L$(OUT) -lfamsa_ref -Wl,-rpath,'$$ORIGIN'

$(HOBJ): $(HERE)ref_refine_harness.cpp
	@mkdir -p $(OBJ)
	$(CXX) $(REFFLAGS) -c $< -o $@
