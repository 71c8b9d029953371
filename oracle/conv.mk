# Test infrastructure for the convolution (tests/test_ref_pin_conv.py).  `ref-if-present` compiles
# the reference's Convolution sources UNMODIFIED, from where they lie in a reference checkout, with
# ref_conv_driver.cu into oracle/_ref/ (git-ignored), against the Caffe-runtime stand-ins
# ref_stub_conv/ (proto messages, blob) ahead of ref_stub_heads/ (layer, filler, cuBLAS gemm / gemv)
# and ref_stub_loss/ (common, the other math helpers).  This is Caffe's own im2col + sgemm engine,
# the convolution the reference's sources define (not its optional cuDNN layer):
#   libmnc_ref_conv.so        caffe-mnc/src/caffe/layers/{conv_layer.{cpp,cu},base_conv_layer.cpp},
#                             caffe-mnc/src/caffe/util/im2col.{cpp,cu}
#   libmnc_ref_conv_nofma.so  the same with nvcc's FMA contraction off (-fmad=false)
REF ?= /root/reference
NVCC ?= nvcc
SRC := $(REF)/caffe-mnc/src/caffe
LAYER_SRCS := $(SRC)/layers/conv_layer.cpp $(SRC)/layers/conv_layer.cu $(SRC)/layers/base_conv_layer.cpp \
              $(SRC)/util/im2col.cpp $(SRC)/util/im2col.cu
STUB_SRCS := ref_stub_heads/math_heads.cu ref_stub_loss/math_functions.cu
STUB := $(STUB_SRCS) $(wildcard ref_stub_conv/*/*.h* ref_stub_conv/*/*/*.h* ref_stub_heads/*/*.h* \
          ref_stub_heads/*/*/*.h* ref_stub_loss/*.h ref_stub_loss/*/*.h* ref_stub_loss/*/*/*.h*)
NVREF := $(NVCC) -gencode arch=compute_90a,code=sm_90a -O2 -w -Xcompiler -fPIC -Iref_stub_conv \
         -Iref_stub_heads -Iref_stub_loss -I$(REF)/caffe-mnc/include -shared

_ref/libmnc_ref_conv.so: ref_conv_driver.cu $(STUB) $(LAYER_SRCS)
	@mkdir -p _ref
	$(NVREF) -o $@ ref_conv_driver.cu $(STUB_SRCS) $(LAYER_SRCS) -lcublas -lcudart

_ref/libmnc_ref_conv_nofma.so: ref_conv_driver.cu $(STUB) $(LAYER_SRCS)
	@mkdir -p _ref
	$(NVREF) -fmad=false -o $@ ref_conv_driver.cu $(STUB_SRCS) $(LAYER_SRCS) -lcublas -lcudart

ref-if-present:
	@if [ -d $(SRC)/layers ]; then $(MAKE) -f conv.mk _ref/libmnc_ref_conv.so _ref/libmnc_ref_conv_nofma.so; fi
