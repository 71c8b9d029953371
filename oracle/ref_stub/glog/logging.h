// oracle/ref_stub -- TEST INFRASTRUCTURE.  glog stand-in: CHECK / LOG come from the stub's
// caffe/common.hpp.
#include "caffe/common.hpp"
