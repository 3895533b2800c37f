# Builds the REFERENCE's MSDeformAttn backward kernels (unmodified .cuh, read from the reference tree) behind a C-ABI
# shim, next to the forward of oracle/Makefile.  Output only into oracle/_ref/ (git-ignored).  Run where the reference
# tree is present:
#     make -C oracle -f backward.mk        (also done by __graft_entry__.build() when the reference tree is present)
REF ?= /root/reference
SRC := $(REF)/third_party/Mask2Former/mask2former/modeling/pixel_decoder/ops/src
NVCC ?= /usr/local/cuda/bin/nvcc
PY ?= python
TORCH_INC := $(shell $(PY) -c "import torch.utils.cpp_extension as c; print(' '.join('-I'+p for p in c.include_paths()))")

_ref/libref_msda_backward.so: ref_msda_backward_host.cu backward.mk $(SRC)/cuda/ms_deform_im2col_cuda.cuh
	mkdir -p _ref
	$(NVCC) -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -lineinfo -shared -Xcompiler -fPIC \
	    -I$(SRC) $(TORCH_INC) -o $@ ref_msda_backward_host.cu -lcudart
