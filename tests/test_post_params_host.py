"""CPU: run-time post-processing settings (b200pose_post_set_params).  For every parameter set, csrc/post_core.h
compiled for the host with those settings, the parameterised C port of pafprocess and the reference's own
pafprocess.cpp compiled with the set's constants give the same candidates, connections and persons, bit for bit, on
the stick figures, the noise maps and 300 fuzz scenarios; the scenarios tell five planted mistakes apart; the range
check refuses every field one step outside its range."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

import post_params_check as ppc
from conftest import ROOT
from oracle import pafprocess_oracle, post_params

SETS = sorted(post_params.SETS)
FP = ctypes.POINTER(ctypes.c_float)


class HostParams(ctypes.Structure):
    _fields_ = post_params.PortParams._fields_


@pytest.fixture(scope="module")
def core(built):
    lib = ctypes.CDLL(os.path.join(ROOT, "build", "libpostparams_host.so"))
    lib.params_process.argtypes = [ctypes.c_int, FP, ctypes.c_int, FP, ctypes.c_long, ctypes.c_long, ctypes.c_long,
                                   ctypes.c_int, ctypes.POINTER(HostParams)]
    for name in ("params_result", "params_cands", "params_conns"):
        getattr(lib, name).restype = FP
    lib.params_num_cands.restype = lib.params_num_conns.restype = ctypes.c_long
    lib.params_check.argtypes = [ctypes.POINTER(HostParams), ctypes.c_char_p, ctypes.c_int]
    return lib


@pytest.fixture(scope="module")
def scen():
    return ppc.scenarios()


def _quads(n, ptr):
    return np.ctypeslib.as_array(ptr, shape=(n * 4,)).reshape(n, 4).copy() if n else np.zeros((0, 4), np.float32)


def host_run(core, params, jl, paf, h, w):
    """(persons [k, 73], candidates, connections) of the host build; params None: the compile-time defaults."""
    prm = ctypes.byref(HostParams(**params)) if params is not None else None
    nh = core.params_process(len(jl), jl.ctypes.data_as(FP), h * 8, paf.ctypes.data_as(FP), 1, w * 38, 38, 3, prm)
    rows = np.ctypeslib.as_array(core.params_result(), shape=(nh * 73,)).reshape(nh, 73).copy() if nh else \
        np.zeros((0, 73), np.float32)
    return rows, _quads(core.params_num_cands(), core.params_cands()), _quads(core.params_num_conns(), core.params_conns())


def port_run(port, jl, paf, h, w):
    rows = ppc.oracle_rows(port, jl, paf, h, w)
    lib = port._lib
    for name in ("port_params_cands", "port_params_conns"):
        getattr(lib, name).restype = FP
    lib.port_params_num_cands.restype = lib.port_params_num_conns.restype = ctypes.c_long
    return rows, _quads(lib.port_params_num_cands(), lib.port_params_cands()), \
        _quads(lib.port_params_num_conns(), lib.port_params_conns())


@pytest.mark.parametrize("name", SETS)
def test_host_core_port_and_reference_agree(name, core, scen):
    params = post_params.params_of(name)
    port = post_params.load_port(name)
    ref = post_params.load_ref(name) if post_params.have_ref(name) else None
    persons = cands = 0
    for key, (jl, paf, h, w) in scen.items():
        got = host_run(core, params, jl, paf, h, w)
        want = port_run(port, jl, paf, h, w)
        for g, wnt, what in zip(got, want, ("persons", "candidates", "connections")):
            assert ppc.same_bits(g, wnt), (name, key, what, g.shape, wnt.shape)
        if ref is not None:
            assert ppc.same_bits(got[0], ppc.oracle_rows(ref, jl, paf, h, w)), (name, key, "reference")
        persons += len(got[0])
        cands += len(got[1])
    print(name, "persons", persons, "candidates", cands, "reference", ref is not None)
    assert persons > 0


def test_reference_builds_exist_where_the_reference_does():
    if not os.path.isdir(os.path.join(post_params.REF, "lib", "pafprocess")) and not all(map(post_params.have_ref, SETS)):
        pytest.skip("no reference sources and no reference builds on this machine")
    assert all(post_params.have_ref(n) for n in SETS)


def test_defaults_equal_the_compile_time_instantiation_and_the_unchanged_port(core, scen):
    """`default` through PostParams == DefaultPostParams (host); the parameterised port with `default` == the port's
    unchanged entry point."""
    params = post_params.params_of("default")
    port, plain = post_params.load_port("default"), pafprocess_oracle.load_port()
    for key, (jl, paf, h, w) in scen.items():
        a, b = host_run(core, params, jl, paf, h, w), host_run(core, None, jl, paf, h, w)
        assert all(ppc.same_bits(x, y) for x, y in zip(a, b)), key
        assert ppc.same_bits(ppc.oracle_rows(port, jl, paf, h, w), ppc.oracle_rows(plain, jl, paf, h, w)), key


MUTANTS = {      # planted mistake -> (text in oracle/pafprocess_params.c, replacement)
    ">= for paf_min_above": ("crit1 > prm->paf_min_above", "crit1 >= prm->paf_min_above"),
    "sample count off by one": ("const int steps = prm->paf_samples;", "const int steps = prm->paf_samples + 1;"),
    "scores / 10 kept": ("(scores / (float)steps)", "(scores / 10.f)"),
    "<= in the part-count prune": ("rows[r * 20 + 19] < (float)prm->min_parts", "rows[r * 20 + 19] <= (float)prm->min_parts"),
    "person score / 18": ("rows[r * 20 + 18] / rows[r * 20 + 19] < prm->min_person_score",
                          "rows[r * 20 + 18] / 18.f < prm->min_person_score"),
}


@pytest.mark.parametrize("mutant", list(MUTANTS))
def test_scenarios_tell_planted_mistakes_apart(mutant, scen, tmp_path):
    src = open(os.path.join(ROOT, "oracle", "pafprocess_params.c")).read()
    old, new = MUTANTS[mutant]
    assert src.count(old) == 1
    path = tmp_path / "pafprocess_params.c"
    path.write_text(src.replace(old, new))
    so = str(tmp_path / "libmutant.so")
    subprocess.run(["gcc", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-I" + os.path.join(ROOT, "oracle"), str(path),
                    "-o", so, "-lm"], check=True)
    for name in SETS:
        good = post_params.load_port(name)
        bad = post_params._Port(so, post_params.params_of(name))
        for key, (jl, paf, h, w) in scen.items():
            if not ppc.same_bits(ppc.oracle_rows(good, jl, paf, h, w), ppc.oracle_rows(bad, jl, paf, h, w)):
                print(mutant, "caught by", name, key)
                return
    pytest.fail("no scenario of any set tells '%s' apart" % mutant)


def test_range_check_refuses_every_field_one_step_outside(core):
    def check(**fields):
        p = post_params.params_of("default")
        p.update(fields)
        msg = ctypes.create_string_buffer(200)
        return core.params_check(ctypes.byref(HostParams(**p)), msg, 200) == 1, msg.value.decode()
    inf, nan = float("inf"), float("nan")
    for fields in ({"paf_samples": 1, "paf_min_above": -1}, {"paf_samples": 1, "paf_min_above": 1},
                   {"paf_samples": 64, "paf_min_above": 64}, {"min_parts": 0}, {"min_parts": 18},
                   {"paf_thresh": -3.4e38, "min_person_score": 3.4e38}):
        assert check(**fields) == (True, ""), fields
    for field, value, extra in (("paf_thresh", inf, {}), ("paf_thresh", -inf, {}), ("paf_thresh", nan, {}),
                                ("paf_samples", 0, {"paf_min_above": 0}), ("paf_samples", 65, {}),
                                ("paf_min_above", -2, {}), ("paf_min_above", 11, {}), ("min_parts", -1, {}),
                                ("min_parts", 19, {}), ("min_person_score", inf, {}), ("min_person_score", nan, {})):
        ok, msg = check(**dict(extra, **{field: value}))
        assert not ok and re.match(field + " must be", msg), (field, value, msg)
