import importlib
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (run with -m gpu on a machine that has one)")


def golden(name):
    return np.load(os.path.join(GOLDEN, name + ".npz"))


def pkg_module(name):
    import _b200_alias
    _b200_alias.load_package()
    return importlib.import_module(_b200_alias.PKG + "." + name)


@pytest.fixture(scope="session")
def built():
    """Everything compiled (no-op when up to date)."""
    import __graft_entry__ as g
    g.build()
    return True


@pytest.fixture(scope="session")
def he_sd():
    from oracle import net_port
    return net_port.he_state_dict(1234)


POST_CASES = {
    "p1": lambda s: s.stick_figures(1, 1)[:2], "p3": lambda s: s.stick_figures(3, 3)[:2],
    "p8": lambda s: s.stick_figures(8, 8)[:2], "p30": lambda s: s.stick_figures(30, 30)[:2],
    "noise0": lambda s: s.noise_maps(0),
    "empty": lambda s: (np.zeros((46, 46, 19), np.float32), np.zeros((46, 46, 38), np.float32)),
    "p5_40x52": lambda s: s.stick_figures(5, 55, h=40, w=52)[:2],
}


def humans_rows_to_dicts(rows):
    """golden `humans` array [k, 1+18*3] -> [(score, {part: (x, y, s)})]"""
    out = []
    for r in rows:
        parts = {p: tuple(float(v) for v in r[1 + 3 * p: 4 + 3 * p]) for p in range(18) if r[1 + 3 * p] >= 0}
        out.append((float(r[0]), parts))
    return out


def assert_humans_equal(got, want, coord_tol=0.0, score_tol=2e-6):
    assert len(got) == len(want), "human count %d vs %d" % (len(got), len(want))
    for i, ((gs, gp), (ws, wp)) in enumerate(zip(got, want)):
        assert sorted(gp) == sorted(wp), "human %d parts differ: %s vs %s" % (i, sorted(gp), sorted(wp))
        for p in gp:
            assert abs(gp[p][0] - wp[p][0]) <= coord_tol and abs(gp[p][1] - wp[p][1]) <= coord_tol, (i, p, gp[p], wp[p])
            assert abs(gp[p][2] - wp[p][2]) <= score_tol, (i, p, gp[p], wp[p])
        assert abs(gs - ws) <= 1e-5, (i, gs, ws)
