# Test infrastructure for the layers' backward passes (tests/test_oracle_backward.py,
# tests/test_ref_pin_backward.py, scripts/bench_roi_backward.py), kept apart from Makefile's
# forward-pass recipes.  `make -f backward.mk` builds the C restatement; `ref-if-present` compiles
# the reference's layer sources UNMODIFIED, from where they lie in a reference checkout, with the
# Backward driver into oracle/_ref/ (git-ignored):
#   libmnc_ref_backward.so        caffe-mnc/src/caffe/layers/{roi_warping,mask_resize,mask_pooling,
#                                 roi_pooling}_layer.{cu,cpp} + ref_backward_driver.cu, against the
#                                 Caffe-runtime stand-in in ref_stub/
#   libmnc_ref_backward_nofma.so  the same with nvcc's FMA contraction off (-fmad=false): the
#                                 feature and mask gradients must equal the C restatement bit for bit
REF ?= /root/reference
NVCC ?= nvcc
LAYERS := $(REF)/caffe-mnc/src/caffe/layers
LAYER_SRCS := $(foreach l,roi_warping mask_resize mask_pooling roi_pooling,$(LAYERS)/$(l)_layer.cu $(LAYERS)/$(l)_layer.cpp)
NVREF := $(NVCC) -gencode arch=compute_90a,code=sm_90a -O2 -w -Xcompiler -fPIC -Iref_stub \
         -I$(REF)/caffe-mnc/include -shared

all: liboracle_backward.so

liboracle_backward.so: mnc_oracle_backward.c
	gcc -O2 -fopenmp -ffp-contract=off -fno-fast-math -shared -fPIC -o $@ $< -lm

_ref/libmnc_ref_backward.so: ref_backward_driver.cu $(wildcard ref_stub/caffe/*.hpp ref_stub/caffe/*/*) $(LAYER_SRCS)
	@mkdir -p _ref
	$(NVREF) -o $@ ref_backward_driver.cu $(LAYER_SRCS) -lcudart

_ref/libmnc_ref_backward_nofma.so: ref_backward_driver.cu $(wildcard ref_stub/caffe/*.hpp ref_stub/caffe/*/*) $(LAYER_SRCS)
	@mkdir -p _ref
	$(NVREF) -fmad=false -o $@ ref_backward_driver.cu $(LAYER_SRCS) -lcudart

ref-if-present:
	@if [ -d $(LAYERS) ]; then $(MAKE) -f backward.mk _ref/libmnc_ref_backward.so _ref/libmnc_ref_backward_nofma.so; fi
