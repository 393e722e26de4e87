"""GPU (-m gpu): run-time post-processing settings (b200pose_post_set_params).  For every parameter set the device
post-processing gives the peaks and person rows of the parameterised C port of pafprocess bit for bit, from host maps
in either layout and from device tensors; the fused entry points post-process with the settings of their post object;
two runs in flight keep their own settings; the defaults set explicitly run exactly what an untouched object runs;
a refused value leaves the object usable, and a loose prune meets human_cap like any other run."""
import numpy as np
import pytest
import torch

import post_params_check as ppc
from conftest import pkg_module
from oracle import post_params, synth

pytestmark = pytest.mark.gpu

SETS = sorted(post_params.SETS)
EDGE = {synth.edge_case_name(*c): c for c in synth.EDGE_CASES}


@pytest.fixture(scope="module")
def eng(built):
    return pkg_module("engine")


@pytest.fixture(scope="module")
def maps():
    """name -> (heat, paf) HWC: the stick figures, the noise maps and the edge maps of oracle/synth.EDGE_CASES."""
    out = {n: ppc.stick_case(n) for n in ppc.STICK_CASES}
    out.update({n: synth.edge_maps(*c) for n, c in EDGE.items()})
    return out


def _want(port, heat, paf):
    jl = ppc.joint_list(heat)
    h, w = heat.shape[:2]
    return jl, (ppc.oracle_rows(port, jl, paf, h, w) if len(jl) else np.zeros((0, 73), np.float32))


def _check(post, i, want, what):
    jl, rows = want
    assert post.status(i) == 0, what
    np.testing.assert_array_equal(post.peaks(i), jl, err_msg=str(what))
    got = post.humans(i)
    assert ppc.same_bits(got, rows), (what, got.shape, rows.shape)
    return len(rows)


@pytest.mark.parametrize("name", SETS)
def test_direct_runs_equal_the_port(name, eng, maps):
    port = post_params.load_port(name)
    want = {k: _want(port, *m) for k, m in maps.items()}
    post = eng.NativePost(0, batch_cap=8, peak_cap=2048, human_cap=2048)
    post.set_params(**post_params.params_of(name))
    assert post.params() == {k: float(np.float32(v)) for k, v in post_params.params_of(name).items()}
    persons = 0
    for k, (heat, paf) in maps.items():            # layout 1 from the host, one image per run
        h, w = heat.shape[:2]
        post.run(np.ascontiguousarray(heat).ctypes.data, np.ascontiguousarray(paf).ctypes.data, False, 1, 1, h, w, 0.1)
        post.sync()
        persons += _check(post, 0, want[k], (name, k, "layout 1"))
    shapes = {}
    for k, (heat, _) in maps.items():
        shapes.setdefault(heat.shape[:2], []).append(k)
    for (h, w), keys in sorted(shapes.items()):     # layout 0 as batches of one shape
        for b in range(0, len(keys), 8):
            ks = keys[b:b + 8]
            heats = np.ascontiguousarray(np.stack([maps[k][0] for k in ks]).transpose(0, 3, 1, 2))
            pafs = np.ascontiguousarray(np.stack([maps[k][1] for k in ks]).transpose(0, 3, 1, 2))
            post.run(heats.ctypes.data, pafs.ctypes.data, False, 0, len(ks), h, w, 0.1)
            post.sync()
            for i, k in enumerate(ks):
                _check(post, i, want[k], (name, k, "layout 0"))
    keys = shapes[(46, 46)][:8]                      # device tensors, layout 1
    heat = torch.from_numpy(np.stack([maps[k][0] for k in keys])).cuda().contiguous()
    paf = torch.from_numpy(np.stack([maps[k][1] for k in keys])).cuda().contiguous()
    torch.cuda.synchronize()
    post.run(heat.data_ptr(), paf.data_ptr(), True, 1, len(keys), 46, 46, 0.1, torch.cuda.current_stream().cuda_stream)
    post.sync()
    for i, k in enumerate(keys):
        _check(post, i, want[k], (name, k, "on device"))
    print(name, "persons", persons)
    assert persons > 0


# ------------------------------------------------------------------------------------------------ fused runs
@pytest.fixture(scope="module")
def net(built, he_sd):
    n = pkg_module("engine").NativeNet(0)
    n.load_state_dict_arrays([v.numpy() for v in he_sd.values()])
    return n


def _debug_maps(pe, n, h, w):
    nat = pkg_module("_native")
    heat = np.empty((n, 19, h, w), np.float32)
    paf = np.empty((n, 38, h, w), np.float32)
    nat.check(nat.lib().b200pose_post_debug_maps(pe.post._h, heat.ctypes.data, heat.size, paf.ctypes.data, paf.size),
              "b200pose_post_debug_maps")
    return heat, paf


@pytest.mark.parametrize("name", ["strict", "loose"])
def test_fused_runs_use_the_settings(name, eng, net):
    """Ragged with flip, uniform with flip, four scales with flip on a ragged batch: each frame's rows and peaks equal
    NativePost.run with the same settings on the maps the fused run averaged (its own extent of the canvas)."""
    nat = pkg_module("_native")
    pe = eng.PoseEngine.from_net(net, mode="bf16", batch_cap=4, peak_cap=1024, human_cap=2048,
                                 post_params=post_params.params_of(name))
    ref = eng.NativePost(0, batch_cap=1, peak_cap=1024, human_cap=2048)
    ref.set_params(**post_params.params_of(name))
    rs = np.random.RandomState(5)
    mixed = [rs.randint(0, 256, s + (3,)).astype(np.uint8) for s in ((90, 123), (70, 150), (96, 97))]
    uniform = rs.randint(0, 256, (2, 90, 123, 3)).astype(np.uint8)
    packed = np.concatenate([f.ravel() for f in mixed])
    shapes = [f.shape[:2] for f in mixed]
    calls = [("ragged flip", shapes, 96, lambda: pe.infer_raw_ragged_async_u8(packed.ctypes.data, False, shapes, 96, 8,
                                                                               0.05, flip=True)),
             ("uniform flip", [(90, 123)] * 2, 96, lambda: pe.infer_raw_async_u8(uniform.ctypes.data, False, 2, 90, 123,
                                                                                 96, 8, 0.05, flip=True)),
             ("4 scales flip", shapes, 64, lambda: pe.infer_raw_multiscale_ragged_async_u8(
                 packed.ctypes.data, False, shapes, (0.5, 1.0, 1.5, 2.0), 64, 8, 0.05, flip=True))]
    persons = 0
    for what, shp, dest, call in calls:
        call()
        rows = [r.copy() for r in pe.fetch_arrays()]
        peaks = [pe.post.peaks(i) for i in range(len(shp))]
        pads = [nat.crop_geometry(h, w, dest, 8)[2] for h, w in shp]
        heat, paf = _debug_maps(pe, len(shp), max(p[0] for p in pads) // 8, max(p[1] for p in pads) // 8)
        for i, (ph, pw) in enumerate(pads):
            h, w = ph // 8, pw // 8
            hh, pp = np.ascontiguousarray(heat[i:i + 1, :, :h, :w]), np.ascontiguousarray(paf[i:i + 1, :, :h, :w])
            ref.run(hh.ctypes.data, pp.ctypes.data, False, 0, 1, h, w, 0.05)
            ref.sync()
            assert ppc.same_bits(rows[i], ref.humans(0)), (name, what, i)
            np.testing.assert_array_equal(peaks[i], ref.peaks(0), err_msg="%s %s %d" % (name, what, i))
            persons += len(rows[i])
    print(name, "fused persons", persons)


# ------------------------------------------------------------------------------------------------ runs in flight
def test_two_runs_in_flight_keep_their_settings(eng, maps):
    port = {n: post_params.load_port(n) for n in ("strict", "loose")}
    keys = [k for k in ("p8", "p30") if k in maps]
    heats = np.ascontiguousarray(np.stack([maps[k][0] for k in keys]))
    pafs = np.ascontiguousarray(np.stack([maps[k][1] for k in keys]))
    post = eng.NativePost(0, batch_cap=2, peak_cap=2048, human_cap=2048)
    tickets = {}
    for name in ("strict", "loose"):
        post.set_params(**post_params.params_of(name))
        post.run(heats.ctypes.data, pafs.ctypes.data, False, 1, len(keys), 46, 46, 0.1)
        tickets[name] = post.last_ticket()
    for name in ("strict", "loose"):
        post.select(tickets[name])
        for i, k in enumerate(keys):
            _, rows = _want(port[name], *maps[k])
            assert ppc.same_bits(post.humans(i), rows), (name, k)
    assert len(_want(port["strict"], *maps["p30"])[1]) != len(_want(port["loose"], *maps["p30"])[1])


def test_explicit_defaults_equal_never_setting_anything(eng, maps):
    heats = np.ascontiguousarray(np.stack([maps[k][0] for k in ("p3", "p8", "p30", "noise0")]))
    pafs = np.ascontiguousarray(np.stack([maps[k][1] for k in ("p3", "p8", "p30", "noise0")]))
    out = []
    for how in ("untouched", "explicit", "restored"):
        post = eng.NativePost(0, batch_cap=4, peak_cap=2048, human_cap=2048)
        if how == "explicit":
            post.set_params(**post_params.params_of("default"))
        elif how == "restored":
            post.set_params(**post_params.params_of("loose"))
            post.set_params()
        post.run(heats.ctypes.data, pafs.ctypes.data, False, 1, 4, 46, 46, 0.1)
        post.sync()
        out.append([(post.humans(i).copy(), post.peaks(i)) for i in range(4)])
    for other in out[1:]:
        for (a, pa), (b, pb) in zip(out[0], other):
            assert ppc.same_bits(a, b) and np.array_equal(pa, pb)


# ------------------------------------------------------------------------------------------------ errors, capacity
def test_refused_values_leave_the_object_usable(eng, maps):
    nat = pkg_module("_native")
    post = eng.NativePost(0, batch_cap=1, peak_cap=2048, human_cap=2048)
    post.set_params(**post_params.params_of("strict"))
    before = post.params()
    for bad in ({"paf_samples": 0}, {"paf_samples": 65}, {"paf_min_above": 21}, {"paf_min_above": -2},
                {"min_parts": 19}, {"min_parts": -1}, {"paf_thresh": float("nan")}, {"min_person_score": float("inf")},
                {"paf_samples": 2 ** 32 + 10}, {"no_such_field": 1}):
        with pytest.raises(nat.B200PoseError, match=list(bad)[0]):
            post.set_params(**dict(post_params.params_of("strict"), **bad))
        assert post.params() == before
    heat, paf = maps["p30"]
    post.run(heat.ctypes.data, paf.ctypes.data, False, 1, 1, 46, 46, 0.1)
    post.sync()
    _check(post, 0, _want(post_params.load_port("strict"), heat, paf), "after refusals")


def test_single_crowd_meets_human_cap(eng, maps):
    """Under `single` (every pair with one positive sample, no prune) a crowd keeps many more persons: with
    human_cap = k - 1 the run sets status bit 8, with human_cap = k it keeps all k, as the oracle's row count says."""
    heat, paf = maps["p30"]
    jl, rows = _want(post_params.load_port("single"), heat, paf)
    k = len(rows)
    assert k > len(_want(post_params.load_port("default"), heat, paf)[1])
    for cap, bits in ((k - 1, 8), (k, 0)):
        post = eng.NativePost(0, batch_cap=1, peak_cap=2048, human_cap=cap)
        post.set_params(**post_params.params_of("single"))
        post.run(heat.ctypes.data, paf.ctypes.data, False, 1, 1, 46, 46, 0.1)
        post.sync()
        assert post.status(0) & 0xF == bits, (cap, post.status(0))
        got = post.humans(0)
        assert len(got) == min(k, cap)
        assert ppc.same_bits(got, rows[:len(got)])
