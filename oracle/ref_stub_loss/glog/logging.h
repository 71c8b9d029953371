// oracle/ref_stub_loss -- TEST INFRASTRUCTURE.  glog stand-in: CHECK / LOG come from the stub's
// caffe/common.hpp.
#include "caffe/common.hpp"
