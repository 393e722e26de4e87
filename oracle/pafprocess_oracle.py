"""ORACLE (test infrastructure only).  ctypes front-ends with the calling convention of the reference's SWIG
module (/root/reference/lib/pafprocess/pafprocess.i:14, pafprocess.h:53-59) for

  * `port`: oracle/pafprocess_port.c (plain-C restatement, always buildable), and
  * `ref` : oracle/_ref/libpafprocess_ref.so = the UNMODIFIED /root/reference/lib/pafprocess/pafprocess.cpp
            compiled by oracle/Makefile (`make ref`; only possible where /root/reference exists; the built .so
            travels to the GPU box).
"""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_FP = ctypes.POINTER(ctypes.c_float)


def build(ref=True):
    subprocess.run(["make", "-s", "-C", _HERE, "all"], check=True)
    if ref and os.path.isdir("/root/reference/lib/pafprocess"):
        subprocess.run(["make", "-s", "-C", _HERE, "ref"], check=True)


class _PafProcess:
    """Mimics the SWIG module object: process_paf(peaks[1,P,5], heat_up[H,W,19], paf_up[H,W,38]) + getters."""

    def __init__(self, path, prefix):
        self._lib = ctypes.CDLL(path)
        f = getattr(self._lib, prefix + "process_paf")
        f.argtypes = [ctypes.c_int] * 3 + [_FP] + [ctypes.c_int] * 3 + [_FP] + [ctypes.c_int] * 3 + [_FP]
        f.restype = ctypes.c_int
        self._process = f
        for name, args, res in [("get_num_humans", [], ctypes.c_int),
                                ("get_part_cid", [ctypes.c_int, ctypes.c_int], ctypes.c_int),
                                ("get_score", [ctypes.c_int], ctypes.c_float),
                                ("get_part_x", [ctypes.c_int], ctypes.c_int),
                                ("get_part_y", [ctypes.c_int], ctypes.c_int),
                                ("get_part_score", [ctypes.c_int], ctypes.c_float)]:
            fn = getattr(self._lib, prefix + name)
            fn.argtypes = args
            fn.restype = res
            setattr(self, name, fn)

    def process_paf(self, peaks, heat, paf):
        for a in (peaks, heat, paf):   # numpy.i IN_ARRAY3 semantics: float32, 3-D, C-contiguous
            if a.dtype != np.float32 or a.ndim != 3:
                raise TypeError("Array of type 'float' with 3 dimensions required")
        peaks, heat, paf = (np.ascontiguousarray(a) for a in (peaks, heat, paf))
        return self._process(*peaks.shape, peaks.ctypes.data_as(_FP), *heat.shape, heat.ctypes.data_as(_FP),
                             *paf.shape, paf.ctypes.data_as(_FP))

    def connections(self, limb):
        """(a int32 [k], b int32 [k], score float32 [k]): the connections the last call chose for `limb`, in the order
        of its greedy loop (pafprocess.cpp:98-124), a and b peak indices within the limb's two parts.  The port only."""
        L = self._lib
        L.port_get_connection.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.POINTER(ctypes.c_int),
                                          ctypes.POINTER(ctypes.c_int), _FP]
        L.port_get_connection.restype = None
        k = L.port_get_num_connections(int(limb))
        a, b, s = np.zeros(k, np.int32), np.zeros(k, np.int32), np.zeros(k, np.float32)
        ia, ib, fs = ctypes.c_int(), ctypes.c_int(), ctypes.c_float()
        for i in range(k):
            L.port_get_connection(int(limb), i, ctypes.byref(ia), ctypes.byref(ib), ctypes.byref(fs))
            a[i], b[i], s[i] = ia.value, ib.value, fs.value
        return a, b, s

    def humans(self, num_parts=18):
        """[(score, {part: (x, y, peak_score, cid)})] in subset order."""
        out = []
        for h in range(self.get_num_humans()):
            parts = {}
            for p in range(num_parts):
                c = int(self.get_part_cid(h, p))
                if c < 0:
                    continue
                parts[p] = (self.get_part_x(c), self.get_part_y(c), float(self.get_part_score(c)), c)
            out.append((float(self.get_score(h)), parts))
        return out


def load_port():
    path = os.path.join(_HERE, "libpafprocess_port.so")
    if not os.path.exists(path):
        build(ref=False)
    return _PafProcess(path, "port_")


def have_ref():
    return os.path.exists(os.path.join(_HERE, "_ref", "libpafprocess_ref.so"))


def load_ref():
    return _PafProcess(os.path.join(_HERE, "_ref", "libpafprocess_ref.so"), "ref_")
