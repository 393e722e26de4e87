// Host build of csrc/fp8_core.h for tests/test_fp8_host.py: the e4m3 quantiser the weight packer uses, the scale exponent
// rule the kernels use, and the K order of the fp8 A fragments.
#include <cstdint>

#include "../../pytorch_realtime_multi-person_pose_estimation_b200/csrc/fp8_core.h"

extern "C" {
void core_e4m3_rn(const float* x, uint8_t* out, long n) {
    for (long i = 0; i < n; ++i) out[i] = b2p::e4m3_rn_bits(x[i]);
}
void core_fp8_exp(const uint32_t* bits, int* out, long n) {
    for (long i = 0; i < n; ++i) out[i] = b2p::fp8_exp_from_amax(bits[i]);
}
int core_k_to_channel(int k) { return b2p::fp8_k_to_channel(k); }
}
