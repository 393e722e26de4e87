"""CPU: the adversarial heat maps of oracle/synth.EDGE_CASES (plateaus, k/16 values, checkerboards, maxima exactly at
the threshold, spikes on every edge row and column, adjacent equal maxima) do what their names say, and the oracle
(nms_port + the C port of pafprocess) reproduces what the reference's own NMS and pafprocess.cpp made of them
(tests/golden/post_edges.npz, written by `python tests/golden/make_golden.py edges`) bit for bit."""
import hashlib

import numpy as np
import pytest

from conftest import assert_humans_equal, golden, humans_rows_to_dicts
from oracle import glue_port, nms_port, pafprocess_oracle, synth

THRESH = 0.1
CASES = {synth.edge_case_name(*c): c for c in synth.EDGE_CASES}


@pytest.fixture(scope="module")
def fixture():
    return golden("post_edges")


@pytest.fixture(scope="module")
def maps():
    return {name: synth.edge_maps(*c) for name, c in CASES.items()}


def test_edge_scenarios_equal_the_golden_inputs(fixture, maps):
    h = hashlib.sha256()
    for name in CASES:
        for a in maps[name]:
            h.update(np.ascontiguousarray(a).tobytes())
    assert h.hexdigest()[:16] == str(fixture["in_digest"]), "oracle/synth.edge_maps drifted from the golden inputs"


def _stats(heat, kind):
    """What a scenario exercises, measured on the oracle: low-res peaks with an equal 4-neighbour, refinements whose
    maximum is attained at two or more up-sampled positions, peaks per edge row / column, pixels exactly at /
    just above the threshold (and how many of them are peaks), peak ids sharing one refined position."""
    h, w = heat.shape[:2]
    st = dict(equal_nb=0, tie_refine=0, at=0, at_peaks=0, above=0, above_max=0, above_peaks=0, shared=0,
              rows={}, cols={})
    at, above = np.float32(THRESH), np.nextafter(np.float32(THRESH), np.float32(np.inf))
    for part in range(18):
        m = np.ascontiguousarray(heat[:, :, part])
        coords = nms_port.find_peaks(THRESH, m)
        peak = np.zeros((h, w), bool)
        peak[coords[:, 1], coords[:, 0]] = True
        st["at"] += int((m == at).sum())
        st["at_peaks"] += int(((m == at) & peak).sum())
        st["above"] += int((m == above).sum())
        st["above_peaks"] += int(((m == above) & peak).sum())
        for x, y in coords:
            v = m[y, x]
            nb = [m[y + dy, x + dx] for dy, dx in ((-1, 0), (1, 0), (0, -1), (0, 1)) if 0 <= y + dy < h and 0 <= x + dx < w]
            st["equal_nb"] += any(u == v for u in nb)
            for r in {0, 1, 2, h - 3, h - 2, h - 1}:
                st["rows"][r] = st["rows"].get(r, 0) + (y == r)
            for c in {0, 1, 2, w - 3, w - 2, w - 1}:
                st["cols"][c] = st["cols"].get(c, 0) + (x == c)
            up = nms_port.upsample8_cubic(m[max(0, y - 2):min(h, y + 3), max(0, x - 2):min(w, x + 3)])
            st["tie_refine"] += int((up == up.max()).sum() >= 2)
        if kind == "threshold":     # every pixel just above the threshold that is >= its neighbours must be a peak
            ge = nms_port.find_peaks(-np.inf, m)
            st["above_max"] += int(sum(m[y, x] == above for x, y in ge))
        jl = nms_port.joint_list_from_nms(nms_port.nms(m[:, :, None], THRESH, 1))
        _, n = np.unique(jl[:, :2], axis=0, return_counts=True)
        st["shared"] += int((n - 1).sum())
    return st


@pytest.mark.parametrize("kind", sorted(synth.EDGE_KINDS))
def test_edge_scenarios_exercise_what_they_claim(kind, maps):
    names = [n for n, c in CASES.items() if c[0] == kind]
    tot = {}
    for name in names:
        st = _stats(maps[name][0], kind)
        for k, v in st.items():
            if isinstance(v, dict):
                continue
            tot[k] = tot.get(k, 0) + v
        c = CASES[name]
        if kind == "border" and min(c[2], c[3]) >= 5:
            assert all(v > 0 for v in st["rows"].values()), (name, st["rows"])
            assert all(v > 0 for v in st["cols"].values()), (name, st["cols"])
            print(name, "peaks on rows", st["rows"], "on columns", st["cols"])
    print(kind, tot)
    assert tot["at_peaks"] == 0                        # `img > thresh`: a pixel exactly at float32(thresh) is no peak
    if kind in ("plateau", "quantised", "twins"):
        assert tot["equal_nb"] > 50
    if kind in ("plateau", "quantised", "checkerboard"):
        assert tot["tie_refine"] > 50
    if kind == "twins":
        assert tot["shared"] > 50
    if kind == "threshold":
        assert tot["at"] > 100 and tot["above"] > 100
        assert tot["above_peaks"] == tot["above_max"] > 100


def test_checkerboard_peak_counts(maps):
    for name, c in CASES.items():
        if c[0] != "checkerboard":
            continue
        heat = maps[name][0]
        h, w = c[2], c[3]
        for part in range(18):
            n = len(nms_port.find_peaks(THRESH, np.ascontiguousarray(heat[:, :, part])))
            assert n in (h * w // 2, (h * w + 1) // 2), (name, part, n)
            if h * w % 2 == 0:
                assert n == h * w // 2


@pytest.mark.parametrize("name", list(CASES))
def test_oracle_equals_reference_golden_on_edge_scenarios(name, fixture, maps):
    heat, paf = maps[name]
    jl = nms_port.joint_list_from_nms(nms_port.nms(heat, THRESH))
    np.testing.assert_array_equal(jl, fixture[name + "_joint_list"])
    jl2, humans = glue_port.paf_to_pose(heat, paf, pafprocess_oracle.load_port(), thresh=THRESH)
    np.testing.assert_array_equal(jl2, jl)
    assert_humans_equal(humans, humans_rows_to_dicts(fixture[name + "_humans"]), score_tol=0.0)
    if pafprocess_oracle.have_ref():      # the reference's own translation unit on the same peaks: identical
        _, href = glue_port.paf_to_pose(heat, paf, pafprocess_oracle.load_ref(), thresh=THRESH)
        assert humans == href
