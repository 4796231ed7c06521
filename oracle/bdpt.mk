# TEST INFRASTRUCTURE ONLY.  Builds
#   oracle/_ref/libbdpt_ref.so   the UNMODIFIED examples/bidir_path_tracer/main.cc (Random, LightSampler, raytrace,
#                                eyeSubpath, lightSubpath, weightMIS, calcG, connectPath) behind bdpt_ref_shim.cc
# -ftrivial-auto-var-init=zero: the light-origin vertex's material, which the reference leaves uninitialised and then
# reads (main.cc:1064, 1203-1204), is zero -- not delta, as the device defines it.  Where the reference tree is absent
# an earlier build is kept.
NANORT_REF ?= /root/reference
CXX ?= g++
FPFLAGS = -O2 -ffp-contract=off -fno-fast-math -ftrivial-auto-var-init=zero
R = $(NANORT_REF)/examples/bidir_path_tracer

all:
	@if [ -f $(R)/main.cc ]; then \
	  mkdir -p _ref && \
	  $(CXX) -std=c++11 $(FPFLAGS) -w -DNANORT_USE_CPP11_FEATURE -fPIC -shared -pthread \
	      -I$(NANORT_REF) -I$(R) -I$(NANORT_REF)/examples/common \
	      -Wl,-Bsymbolic -o _ref/libbdpt_ref.so bdpt_ref_shim.cc $(R)/tiny_obj_loader.cc && \
	  echo "built oracle/_ref/libbdpt_ref.so from $(R)/main.cc"; \
	else \
	  echo "$(R)/main.cc not present: keeping prebuilt oracle/_ref/libbdpt_ref.so (if any)"; \
	fi

.PHONY: all
