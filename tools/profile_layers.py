#!/usr/bin/env python
"""Per-launch device time and algorithmic TFLOP/s of one bf16 forward (CUDA events around every launch through
b200pose_net_profile).  Usage on an H100: python tools/profile_layers.py [batch]"""
import ctypes
import importlib
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import _b200_alias  # noqa: E402

_b200_alias.load_package()
import torch  # noqa: E402

engine = importlib.import_module(_b200_alias.PKG + ".engine")
nat = importlib.import_module(_b200_alias.PKG + "._native")
syn = importlib.import_module(_b200_alias.PKG + ".synthetic")

NAMES = (["conv1_1 (cuda cores)", "conv1_2+pool", "conv2_1", "conv2_2+pool", "conv3_1", "conv3_2", "conv3_3", "conv3_4+pool",
          "conv4_1", "conv4_2", "conv4_3_CPM", "conv4_4_CPM"] +
         ["conv5_%d_CPM L1|L2" % i for i in range(1, 6)] +
         ["Mconv%d_stage%d L1|L2" % (i, s) for s in range(2, 7) for i in range(1, 8)])


def main():
    batch = int(sys.argv[1]) if len(sys.argv) > 1 else 32
    net = engine.NativeNet(0)
    net.load_state_dict_arrays(syn.he_state_arrays(1234))
    x = (torch.rand((batch, 3, 368, 368), generator=torch.Generator().manual_seed(1)) - 0.5).cuda()
    st = torch.cuda.current_stream().cuda_stream
    for _ in range(3):
        net.forward_ptr(x.data_ptr(), True, batch, 368, 368, 0, [0] * 12, True, st)
    torch.cuda.synchronize()
    cap = 64
    ms, fl = (ctypes.c_float * cap)(), (ctypes.c_double * cap)()
    acc = [0.0] * cap
    reps = 5
    for _ in range(reps):
        n = nat.lib().b200pose_net_profile(net._h, ms, fl, cap, ctypes.c_void_p(st))
        assert n > 0
        for i in range(n):
            acc[i] += ms[i] / reps
    tot = sum(acc[:n])
    print("batch %d, 368x368, bf16; %d launches; total %.3f ms (%.1f frames/s net only)" % (batch, n, tot, batch / tot * 1e3))
    print("%-28s %9s %9s %7s" % ("launch", "ms", "TFLOP/s", "share"))
    for i in range(n):
        print("%-28s %9.4f %9.1f %6.1f%%" % (NAMES[i], acc[i], fl[i] / acc[i] * 1e-9, 100 * acc[i] / tot))
    tc_ms = sum(acc[1:n])
    tc_fl = sum(fl[i] for i in range(1, n))
    print("tensor-core launches: %.3f ms, %.1f TFLOP/s aggregate" % (tc_ms, tc_fl / tc_ms * 1e-9))


if __name__ == "__main__":
    main()
