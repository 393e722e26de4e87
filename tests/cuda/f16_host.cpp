// Host build of csrc/f16_core.h for tests/test_fp16_host.py: the binary16 rounding the fp16 weight packer uses.
#include <cstdint>

#include "../../pytorch_realtime_multi-person_pose_estimation_b200/csrc/f16_core.h"

extern "C" {
void core_f16_rn(const float* x, uint16_t* out, long n) {
    for (long i = 0; i < n; ++i) out[i] = b2p::f16_rn_bits(x[i]);
}
}
