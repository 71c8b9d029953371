# Test infrastructure for the head layers (tests/test_ref_pin_heads.py).  `ref-if-present` compiles
# the reference's head-layer sources UNMODIFIED, from where they lie in a reference checkout, with
# ref_heads_driver.cu into oracle/_ref/ (git-ignored), against the Caffe-runtime stand-ins
# ref_stub_heads/ (proto messages, layer parameters, filler, cuBLAS gemm / gemv) ahead of
# ref_stub_loss/ (blob, common, the other math helpers):
#   libmnc_ref_heads.so        caffe-mnc/src/caffe/layers/{inner_product,pooling,relu,sigmoid}_layer
#                              .{cpp,cu}, neuron_layer.cpp
#   libmnc_ref_heads_nofma.so  the same with nvcc's FMA contraction off (-fmad=false)
REF ?= /root/reference
NVCC ?= nvcc
LAYERS := $(REF)/caffe-mnc/src/caffe/layers
LAYER_SRCS := $(foreach l,inner_product pooling relu sigmoid,$(LAYERS)/$(l)_layer.cu $(LAYERS)/$(l)_layer.cpp) \
              $(LAYERS)/neuron_layer.cpp
STUB_SRCS := ref_stub_heads/math_heads.cu ref_stub_loss/math_functions.cu
STUB := $(STUB_SRCS) $(wildcard ref_stub_heads/*/*.h* ref_stub_heads/*/*/*.h* ref_stub_loss/*.h ref_stub_loss/*/*.h* ref_stub_loss/*/*/*.h*)
NVREF := $(NVCC) -gencode arch=compute_90a,code=sm_90a -O2 -w -Xcompiler -fPIC -Iref_stub_heads \
         -Iref_stub_loss -I$(REF)/caffe-mnc/include -shared

_ref/libmnc_ref_heads.so: ref_heads_driver.cu $(STUB) $(LAYER_SRCS)
	@mkdir -p _ref
	$(NVREF) -o $@ ref_heads_driver.cu $(STUB_SRCS) $(LAYER_SRCS) -lcublas -lcudart

_ref/libmnc_ref_heads_nofma.so: ref_heads_driver.cu $(STUB) $(LAYER_SRCS)
	@mkdir -p _ref
	$(NVREF) -fmad=false -o $@ ref_heads_driver.cu $(STUB_SRCS) $(LAYER_SRCS) -lcublas -lcudart

ref-if-present:
	@if [ -d $(LAYERS) ]; then $(MAKE) -f heads.mk _ref/libmnc_ref_heads.so _ref/libmnc_ref_heads_nofma.so; fi
