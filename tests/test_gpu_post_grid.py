"""GPU (-m gpu): the two work-queue kernels of the device post-processing, limb_score_kernel and range_sort_kernel, give
the same results at every grid size.  Both take their work from a global cursor, so a block may score items of several
limbs and images and sort several ranges one after the other; at the default grids and on small scenarios nearly every
block takes one group and exits, and the paths that carry state from one grab to the next never run.

Every scenario of tests/post_grid_check.py runs once at the default grids and must equal the oracle (nms_port, and the
C port of pafprocess with its connections).  It is then rerun at score grids {1, 2, 3, 7, S - 1, S, 12 S} and sort
grids {1, 2, 3, 7, S - 1, 6 S} (S = SM count), the other grid at its default, and must equal the default run bit for
bit: peak rows, the connections of every (image, limb), person rows, status words and the sticky accumulator."""
import numpy as np
import pytest
import torch

import post_grid_check as pgc
import post_params_check as ppc
from conftest import ROOT, pkg_module
from oracle import pafprocess_oracle, post_params

pytestmark = pytest.mark.gpu

SCORE_GRIDS = ("1", "2", "3", "7", "S-1", "S", "12S")
SORT_GRIDS = ("1", "2", "3", "7", "S-1", "6S")
SCENARIOS = pgc.scenarios()


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _blocks(g):
    s = _sms()
    return {"S-1": s - 1, "S": s, "12S": 12 * s, "6S": 6 * s}.get(g) or int(g)


@pytest.fixture(scope="module")
def eng(built):
    return pkg_module("engine")


@pytest.fixture(scope="module")
def post(eng):
    p = eng.NativePost(0, batch_cap=5, peak_cap=2048, human_cap=2048)
    yield p
    p.set_grids(0, 0)


def _run(post, images, layout, params, grids=None):
    """One batch at the given (score, sort) grids (None: the object's own, not touched); returns everything the run
    decided, per image."""
    heats, pafs = np.stack([im[0] for im in images]), np.stack([im[1] for im in images])
    n, h, w = heats.shape[:3]
    if layout == 0:
        heats, pafs = heats.transpose(0, 3, 1, 2), pafs.transpose(0, 3, 1, 2)
    heats, pafs = np.ascontiguousarray(heats, np.float32), np.ascontiguousarray(pafs, np.float32)
    post.set_params(**(post_params.params_of(params) if params else {}))
    post.status_accum(reset=True)
    if grids is not None:
        post.set_grids(*grids)
    try:
        post.run(heats.ctypes.data, pafs.ctypes.data, False, layout, n, h, w, pgc.THRESH)
        post.sync()
    finally:
        if grids is not None:
            post.set_grids(0, 0)
    return {"status": [post.status(i) for i in range(n)], "acc": post.status_accum(reset=True),
            "peaks": [post.peaks(i) for i in range(n)], "humans": [post.humans(i).copy() for i in range(n)],
            "conns": [[post.connections(i, l) for l in range(19)] for i in range(n)]}


def _assert_same(got, want, what):
    assert got["status"] == want["status"] and got["acc"] == want["acc"], what
    for i, (g, w) in enumerate(zip(got["peaks"], want["peaks"])):
        assert ppc.same_bits(g, w), (what, "peaks", i)
    for i, (g, w) in enumerate(zip(got["humans"], want["humans"])):
        assert ppc.same_bits(g, w), (what, "persons", i, g.shape, w.shape)
    for i, (gi, wi) in enumerate(zip(got["conns"], want["conns"])):
        for l, (g, w) in enumerate(zip(gi, wi)):
            assert len(g[0]) == len(w[0]) and np.array_equal(g[0], w[0]) and np.array_equal(g[1], w[1]) \
                and ppc.same_bits(g[2], w[2]), (what, "connections of image %d limb %d" % (i, l), len(g[0]), len(w[0]))


_DEFAULT = {}


def _default(post, name):
    if name not in _DEFAULT:
        _DEFAULT[name] = _run(post, *SCENARIOS[name])
    return _DEFAULT[name]


@pytest.mark.parametrize("name", list(SCENARIOS))
def test_default_grids_equal_the_oracle(name, post):
    images, _, params = SCENARIOS[name]
    port = post_params.load_port(params) if params else pafprocess_oracle.load_port()
    got = _default(post, name)
    assert got["status"] == [0] * len(images) and got["acc"] == 0
    conns = 0
    for i, (heat, paf) in enumerate(images):
        jl = ppc.joint_list(heat)
        np.testing.assert_array_equal(got["peaks"][i], jl, err_msg="%s image %d" % (name, i))
        rows = ppc.oracle_rows(port, jl, paf, *heat.shape[:2]) if len(jl) else np.zeros((0, 73), np.float32)
        assert ppc.same_bits(got["humans"][i], rows), (name, i, got["humans"][i].shape, rows.shape)
        for l in range(19):
            a, b, s = port.connections(l) if len(jl) else (np.zeros(0, np.int32),) * 2 + (np.zeros(0, np.float32),)
            ga, gb, gs = got["conns"][i][l]
            assert np.array_equal(ga, a) and np.array_equal(gb, b) and ppc.same_bits(gs, s), (name, i, l)
            conns += len(a)
    assert conns > 0, name
    print(name, "connections", conns)


@pytest.mark.parametrize("grid", SCORE_GRIDS)
@pytest.mark.parametrize("name", list(SCENARIOS))
def test_score_grid(name, grid, post):
    want = _default(post, name)
    _assert_same(_run(post, *SCENARIOS[name], grids=(_blocks(grid), 0)), want, (name, "score grid", grid))


@pytest.mark.parametrize("grid", SORT_GRIDS)
@pytest.mark.parametrize("name", list(SCENARIOS))
def test_sort_grid(name, grid, post):
    want = _default(post, name)
    _assert_same(_run(post, *SCENARIOS[name], grids=(0, _blocks(grid))), want, (name, "sort grid", grid))


def test_scenarios_reach_the_queue_shapes():
    """On this device: the noise batch has more groups than the largest score grid, so blocks loop at every grid."""
    counts = [pgc.part_counts(h) for h, _ in SCENARIOS["noise46"][0]]
    assert len(pgc.groups(pgc.work_items(counts))) > 12 * _sms()


def test_largest_sorts_at_grid_2(eng):
    """The status-bit-2 boundary scene (8 Mi - 130 Ki candidate pairs, two 4 Mi sorts) at score grid 2 and at sort
    grid 2: identical to its default run, which equals the oracle."""
    post = eng.NativePost(0, batch_cap=1, peak_cap=2048, human_cap=256)
    images = [pgc.bit2_scene()]
    want = _run(post, images, 1, None)
    heat, paf = images[0]
    jl = ppc.joint_list(heat)
    port = pafprocess_oracle.load_port()
    assert want["status"] == [0]
    np.testing.assert_array_equal(want["peaks"][0], jl)
    assert ppc.same_bits(want["humans"][0], ppc.oracle_rows(port, jl, paf, 64, 64))
    for l in range(19):
        a, b, s = port.connections(l)
        assert np.array_equal(want["conns"][0][l][0], a) and np.array_equal(want["conns"][0][l][1], b)
        assert ppc.same_bits(want["conns"][0][l][2], s)
    for grids in ((2, 0), (0, 2)):
        _assert_same(_run(post, images, 1, None, grids=grids), want, ("bit-2 scene", grids))


@pytest.mark.parametrize("grid", ("1", "7", "6S"))
def test_debug_sort_at_sort_grid(grid, eng):
    """The 162 key sets of the device sort test through b200pose_post_debug_sort at sort grid 1, 7 and 6 S: the
    sequential restatement of std::sort, ties included."""
    import ctypes
    import os
    nat = pkg_module("_native")
    host = ctypes.CDLL(os.path.join(ROOT, "build", "libpostcore_host.so"))
    U = ctypes.POINTER(ctypes.c_uint64)
    host.core_seq_sort.argtypes = [U, ctypes.c_int, U]
    post = eng.NativePost(0, batch_cap=1, peak_cap=64, human_cap=16)
    post.set_grids(0, _blocks(grid))
    for hi in pgc.sort_inputs():
        n = len(hi)
        keys = (hi.astype(np.uint64) << np.uint64(32)) | np.arange(n, dtype=np.uint64)
        want, got = np.zeros(n, np.uint64), np.zeros(n, np.uint64)
        host.core_seq_sort(keys.ctypes.data_as(U), n, want.ctypes.data_as(U))
        nat.check(nat.lib().b200pose_post_debug_sort(post._h, keys.ctypes.data, n, got.ctypes.data), "debug_sort")
        bad = np.nonzero(got != want)[0]
        assert bad.size == 0, "grid %s n=%d: first mismatch at %d (%d wrong)" % (grid, n, bad[0], bad.size)


def test_fused_infer_u8_at_grid_1(eng, he_sd):
    """b200pose_infer_u8, three frames in bf16: at score grid 1 and sort grid 1 the same persons, peaks and
    connections as at the defaults."""
    net = eng.NativeNet(0)
    net.load_state_dict_arrays([v.numpy() for v in he_sd.values()])
    pe = eng.PoseEngine.from_net(net, mode="bf16", batch_cap=3, peak_cap=1024, human_cap=1024)
    frames = np.random.RandomState(9).randint(0, 256, (3, 96, 128, 3)).astype(np.uint8)
    out = []
    for grids in ((0, 0), (1, 1), (0, 0)):
        pe.post.set_grids(*grids)
        pe.infer_async_u8(frames.ctypes.data, False, 3, 96, 128)
        rows = [r.copy() for r in pe.fetch_arrays()]
        out.append({"rows": rows, "peaks": [pe.post.peaks(i) for i in range(3)],
                    "conns": [[pe.post.connections(i, l) for l in range(19)] for i in range(3)]})
    pe.post.set_grids(0, 0)
    assert sum(len(c[0]) for ci in out[0]["conns"] for c in ci) > 0
    for other in out[1:]:
        for i in range(3):
            assert ppc.same_bits(other["rows"][i], out[0]["rows"][i]), i
            assert ppc.same_bits(other["peaks"][i], out[0]["peaks"][i]), i
            for l in range(19):
                for g, w in zip(other["conns"][i][l], out[0]["conns"][i][l]):
                    assert len(g) == len(w) and ppc.same_bits(g.view(np.float32), w.view(np.float32)), (i, l)


def test_set_grids_refusals_leave_the_object_usable(eng):
    """Refused grids name the argument and change nothing; after set_grids(0, 0) a run equals one made before any
    override was set."""
    nat = pkg_module("_native")
    post = eng.NativePost(0, batch_cap=3, peak_cap=2048, human_cap=2048)
    images, layout, _ = SCENARIOS["crossing46x46_l1"]
    before = _run(post, images, layout, None)
    for bad, field in (((-1, 0), "score_blocks"), ((65536, 0), "score_blocks"), ((0, -1), "sort_blocks"),
                       ((0, 65536), "sort_blocks"), ((2 ** 32 + 1, 0), "score_blocks")):
        with pytest.raises(nat.B200PoseError, match=field):
            post.set_grids(*bad)
        _assert_same(_run(post, images, layout, None, grids=(0, 0)), before, ("after refusal", bad))
    post.set_grids(1, 65535)
    post.set_grids(0, 0)
    heats = np.ascontiguousarray(np.stack([im[0] for im in images]))
    pafs = np.ascontiguousarray(np.stack([im[1] for im in images]))
    post.status_accum(reset=True)
    post.run(heats.ctypes.data, pafs.ctypes.data, False, layout, len(images), 46, 46, pgc.THRESH)
    post.sync()
    for i in range(len(images)):
        assert ppc.same_bits(post.humans(i), before["humans"][i])
        assert ppc.same_bits(post.peaks(i), before["peaks"][i])
        for l in range(19):
            assert all(np.array_equal(g, w) for g, w in zip(post.connections(i, l), before["conns"][i][l]))
