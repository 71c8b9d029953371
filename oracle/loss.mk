# Test infrastructure for the loss layers (tests/test_ref_pin_loss.py, scripts/bench_losses.py).
# `ref-if-present` compiles the reference's loss-layer sources UNMODIFIED, from where they lie in a
# reference checkout, with ref_loss_driver.cu into oracle/_ref/ (git-ignored), against the
# Caffe-runtime stand-in in ref_stub_loss/ (which also provides the cuBLAS math helpers):
#   libmnc_ref_loss.so        caffe-mnc/src/caffe/layers/{softmax_loss,smooth_L1_loss,
#                             sigmoid_cross_entropy_loss,accuracy,loss,softmax,sigmoid,neuron}_layer
#                             .{cpp,cu}
#   libmnc_ref_loss_nofma.so  the same with nvcc's FMA contraction off (-fmad=false)
REF ?= /root/reference
NVCC ?= nvcc
LAYERS := $(REF)/caffe-mnc/src/caffe/layers
LAYER_SRCS := $(foreach l,softmax_loss smooth_L1_loss sigmoid_cross_entropy_loss softmax sigmoid,$(LAYERS)/$(l)_layer.cu $(LAYERS)/$(l)_layer.cpp) \
              $(foreach l,accuracy loss neuron,$(LAYERS)/$(l)_layer.cpp)
STUB := ref_stub_loss/math_functions.cu $(wildcard ref_stub_loss/*.h ref_stub_loss/*/*.h* ref_stub_loss/*/*/*.h*)
NVREF := $(NVCC) -gencode arch=compute_90a,code=sm_90a -O2 -w -Xcompiler -fPIC -Iref_stub_loss \
         -I$(REF)/caffe-mnc/include -shared

_ref/libmnc_ref_loss.so: ref_loss_driver.cu $(STUB) $(LAYER_SRCS)
	@mkdir -p _ref
	$(NVREF) -o $@ ref_loss_driver.cu ref_stub_loss/math_functions.cu $(LAYER_SRCS) -lcublas -lcudart

_ref/libmnc_ref_loss_nofma.so: ref_loss_driver.cu $(STUB) $(LAYER_SRCS)
	@mkdir -p _ref
	$(NVREF) -fmad=false -o $@ ref_loss_driver.cu ref_stub_loss/math_functions.cu $(LAYER_SRCS) -lcublas -lcudart

ref-if-present:
	@if [ -d $(LAYERS) ]; then $(MAKE) -f loss.mk _ref/libmnc_ref_loss.so _ref/libmnc_ref_loss_nofma.so; fi
