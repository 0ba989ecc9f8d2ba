# Test infrastructure only.  Builds
#   _ref/libinfluence_ref.so : the reference's UNMODIFIED influence-function kernels
#                              (influence_function.cu, compiled where it lies under $(REF), never copied)
#                              for sm_90a, exporting the host launchers cudakernel_hessian,
#                              cudakernel_d_solutions and cudakernel_d_residuals (device pointers in).
# Only the GPU tests of calculate_diagnostics_gpu (tests/test_gpu_diagnostics.py) load it.  nvcc's static
# cudart: the library needs nothing but libc.  Without the reference sources a prebuilt _ref/ is kept.
REF      ?= /root/reference
DIRAC    := $(REF)/src/lib/Dirac
RADIO    := $(REF)/src/lib/Radio

all:
	@if [ -f "$(RADIO)/influence_function.cu" ]; then $(MAKE) --no-print-directory -f influence.mk _ref/libinfluence_ref.so; \
	 else echo "oracle: $(REF) absent, keeping prebuilt _ref/libinfluence_ref.so (if any)"; fi

_ref/libinfluence_ref.so: $(RADIO)/influence_function.cu
	@mkdir -p _ref
	nvcc -gencode arch=compute_90a,code=sm_90a -DHAVE_CUDA -Xcompiler -fPIC -shared -I$(RADIO) -I$(DIRAC) -o $@ $<

.PHONY: all
