"""ORACLE (test infrastructure only).  pafprocess with run-time settings, for the product's b200pose_post_set_params:

  * `load_port(params)`: oracle/pafprocess_params.c, the plain-C port with the five constants of the reference's
    pafprocess.h:7-13 as arguments (always buildable);
  * `load_ref(name)`   : oracle/_ref/<name>/libpafprocess_ref.so, the UNMODIFIED reference pafprocess.cpp compiled with
    the constants of parameter set `name` substituted into a copy of its header (oracle/params.mk; only possible where
    the reference exists, the built .so files travel to the GPU box).

Both return objects with the SWIG module's calling convention, for glue_port.paf_to_pose.
"""
import ctypes
import os
import subprocess

import numpy as np

from .pafprocess_oracle import _PafProcess

_HERE = os.path.dirname(os.path.abspath(__file__))
REF = "/root/reference"
FIELDS = ("paf_thresh", "paf_samples", "paf_min_above", "min_parts", "min_person_score")
# name -> (paf_thresh, paf_samples, paf_min_above, min_parts, min_person_score); the values are written into the
# reference header as they are spelled here, and reach the port and the product as the same float32 / int values
SETS = {
    "default": ("0.05", 10, 6, 4, "0.3"),
    "strict": ("0.1", 20, 15, 5, "0.4"),
    "loose": ("-0.02", 5, 2, 2, "0.1"),
    "single": ("0.05", 1, 0, 0, "-1"),
    "wide": ("0.05", 64, 48, 4, "0.3"),
}


def params_of(name):
    """The set as a dict of the product's field names (NativePost.set_params(**params_of(name)))."""
    return {f: (float(v) if isinstance(v, str) else v) for f, v in zip(FIELDS, SETS[name])}


class PortParams(ctypes.Structure):
    _fields_ = [("paf_thresh", ctypes.c_float), ("paf_samples", ctypes.c_int), ("paf_min_above", ctypes.c_int),
                ("min_parts", ctypes.c_int), ("min_person_score", ctypes.c_float)]


def build(ref=True):
    subprocess.run(["make", "-s", "-C", _HERE, "-f", "params.mk", "port"], check=True)
    if ref and os.path.isdir(os.path.join(REF, "lib", "pafprocess")):
        for name, (t, n, k, m, s) in SETS.items():
            subprocess.run(["make", "-s", "-C", _HERE, "-f", "params.mk", "ref-set", "REF=" + REF, "SET=" + name,
                            "PAF_THRESH=%s" % t, "PAF_SAMPLES=%d" % n, "PAF_MIN_ABOVE=%d" % k, "MIN_PARTS=%d" % m,
                            "MIN_PERSON_SCORE=%s" % s], check=True)


class _Port(_PafProcess):
    """The parameterised port with its settings bound: process_paf(peaks, heat_up, paf_up) uses them."""

    def __init__(self, path, params):
        super().__init__(path, "port_")
        self.params = PortParams(**params)
        f = self._lib.port_process_paf_params
        f.argtypes = list(self._process.argtypes) + [ctypes.POINTER(PortParams)]
        f.restype = ctypes.c_int
        bound = self.params
        self._process = lambda *a: f(*a, ctypes.byref(bound))

    def connections(self, limb):
        """As the port's, from the (limb, a, b, score) quads port_process_paf_params records."""
        L = self._lib
        L.port_params_num_conns.restype = ctypes.c_long
        L.port_params_conns.restype = ctypes.POINTER(ctypes.c_float)
        n = int(L.port_params_num_conns())
        q = np.ctypeslib.as_array(L.port_params_conns(), (n, 4)).copy() if n else np.zeros((0, 4), np.float32)
        q = q[q[:, 0] == limb]
        return q[:, 1].astype(np.int32), q[:, 2].astype(np.int32), np.ascontiguousarray(q[:, 3])


def port_path():
    return os.path.join(_HERE, "libpafprocess_params.so")


def load_port(params=None):
    """params: a dict of FIELDS (missing fields: the reference's constants) or a set name."""
    if not os.path.exists(port_path()):
        build(ref=False)
    p = params_of("default")
    p.update(params_of(params) if isinstance(params, str) else (params or {}))
    return _Port(port_path(), p)


def have_ref(name):
    return os.path.exists(os.path.join(_HERE, "_ref", name, "libpafprocess_ref.so"))


def load_ref(name):
    return _PafProcess(os.path.join(_HERE, "_ref", name, "libpafprocess_ref.so"), "ref_")
