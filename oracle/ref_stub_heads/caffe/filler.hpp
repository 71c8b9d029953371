// oracle/ref_stub_heads -- TEST INFRASTRUCTURE.  Stand-in for caffe/filler.hpp: the driver writes
// the parameters after SetUp, so a filler leaves the blob as it is.
#ifndef MNC_REF_STUB_HEADS_FILLER_HPP_
#define MNC_REF_STUB_HEADS_FILLER_HPP_
#include "caffe/blob.hpp"
#include "caffe/proto/caffe.pb.h"

namespace caffe {
template <typename Dtype>
class Filler {
 public:
  void Fill(Blob<Dtype>*) {}
};
template <typename Dtype>
Filler<Dtype>* GetFiller(const FillerParameter&) { return new Filler<Dtype>(); }
}  // namespace caffe
#endif
