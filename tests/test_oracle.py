"""CPU: pins the oracle (CPU restatements under oracle/) against golden vectors produced by the unmodified
reference (tests/golden/make_golden.py) and against the compiled reference pafprocess.cpp."""
import hashlib
import itertools

import numpy as np
import pytest
import torch

from conftest import POST_CASES, assert_humans_equal, golden, humans_rows_to_dicts
from oracle import glue_port, net_exact, net_port, nms_port, pafprocess_oracle, synth


def _digest(*arrays):
    h = hashlib.sha256()
    for a in arrays:
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()[:16]


@pytest.mark.parametrize("name", ["net_64", "net_368"])
def test_exact_order_network_is_pinned_to_the_reference(name, he_sd):
    """oracle/conv_exact.c (fp32 fused multiply-adds in a defined order) vs the output of the unmodified reference
    module: a different but equally valid fp32 summation order, so the two agree to a few 1e-5 on O(1) maps."""
    g = golden(name)
    hw, seed = int(g["hw"]), int(g["seed"])
    x = torch.rand((1, 3, hw, hw), generator=torch.Generator().manual_seed(seed)) - 0.5
    (paf, heat), saved = net_exact.forward(he_sd, x.numpy())
    assert len(saved) == 12 and paf.shape == g["paf"].shape
    assert np.abs(paf - g["paf"]).max() < 1e-4 and np.abs(heat - g["heat"]).max() < 1e-4
    np.testing.assert_allclose([float(np.abs(t).max()) for t in saved], g["stage_absmax"], rtol=1e-4)


def test_exact_order_network_is_deterministic_and_thread_count_independent(he_sd, monkeypatch):
    x = (torch.rand((2, 3, 40, 56), generator=torch.Generator().manual_seed(2)) - 0.5).numpy()
    _, a = net_exact.forward(he_sd, x)
    monkeypatch.setenv("ORACLE_THREADS", "1")
    _, b = net_exact.forward(he_sd, x)
    for u, v in zip(a, b):
        np.testing.assert_array_equal(u, v)
    # image rows of a batch are independent
    _, c = net_exact.forward(he_sd, x[1:2])
    np.testing.assert_array_equal(c[-1][0], a[-1][1])


@pytest.mark.parametrize("name", ["net_64", "net_368"])
def test_net_port_matches_reference_module(name, he_sd):
    g = golden(name)
    hw, seed = int(g["hw"]), int(g["seed"])
    x = torch.rand((1, 3, hw, hw), generator=torch.Generator().manual_seed(seed)) - 0.5
    assert _digest(x.numpy()) == str(g["x_digest"]), "input regeneration drifted"
    with torch.no_grad():
        (paf, heat), saved = net_port.forward(he_sd, x)
    assert len(saved) == 12
    # same torch ops in the same order as the reference module -> identical up to oneDNN blocking choices
    assert np.abs(paf.numpy() - g["paf"]).max() < 1e-5
    assert np.abs(heat.numpy() - g["heat"]).max() < 1e-5
    np.testing.assert_allclose([float(t.abs().max()) for t in saved], g["stage_absmax"], rtol=1e-5)
    np.testing.assert_allclose(np.stack([t.numpy().reshape(-1)[::13][:64] for t in saved]), g["stage_sample"], atol=1e-5)
    assert float(paf.abs().max()) > 0.5          # non-vacuous: He weights give O(1) outputs


def test_state_dict_spec_is_the_reference_layout():
    spec = net_port.state_dict_spec()
    assert len(spec) == 184
    assert sum(int(np.prod(s)) for s in spec.values()) == 52311446      # SURVEY.md N1
    assert list(spec)[:2] == ["model0.0.weight", "model0.0.bias"] and list(spec)[-1] == "model6_2.12.bias"
    assert spec["model2_1.0.weight"] == (128, 185, 7, 7) and spec["model1_2.8.weight"] == (19, 512, 1, 1)


def test_get_outputs_and_flip_merge(he_sd):
    g = golden("get_outputs_200x230")
    img = np.random.RandomState(0).randint(0, 256, (200, 230, 3)).astype(np.uint8)
    assert _digest(img) == str(g["img_digest"])
    paf, heat, scale = glue_port.get_outputs(img, he_sd, "rtpose")
    assert paf.shape == g["paf"].shape == (46, 53, 38) and abs(scale - float(g["scale"])) < 1e-12
    assert np.abs(paf - g["paf"]).max() < 1e-5 and np.abs(heat - g["heat"]).max() < 1e-5
    f = golden("flip_merge")
    nh, fh = np.random.RandomState(1).rand(6, 5, 19).astype(np.float32), np.random.RandomState(2).rand(6, 5, 19).astype(np.float32)
    npf, fpf = np.random.RandomState(3).rand(6, 5, 38).astype(np.float32), np.random.RandomState(4).rand(6, 5, 38).astype(np.float32)
    ap, ah = glue_port.handle_paf_and_heat(nh, fh, npf, fpf)
    np.testing.assert_array_equal(ap, f["avg_paf"])
    np.testing.assert_array_equal(ah, f["avg_heat"])


def test_bicubic_is_bit_exact_with_opencv_native_path():
    import cv2
    rs = np.random.RandomState(0)
    prev = cv2.ipp.useIPP()
    try:
        for (h, w) in itertools.product([3, 4, 5], [3, 4, 5]):
            for _ in range(4):
                p = rs.rand(h, w).astype(np.float32)
                mine = nms_port.upsample8_cubic(p)
                cv2.ipp.setUseIPP(False)     # OpenCV's own resize.cpp arithmetic
                native = cv2.resize(p, None, fx=8, fy=8, interpolation=cv2.INTER_CUBIC)
                cv2.ipp.setUseIPP(prev)      # the build default (IPP): proprietary arithmetic, a few ulp away
                default = cv2.resize(p, None, fx=8, fy=8, interpolation=cv2.INTER_CUBIC)
                np.testing.assert_array_equal(mine, native)
                assert np.abs(mine - default).max() <= 5e-7
                assert mine.argmax() == default.argmax()
    finally:
        cv2.ipp.setUseIPP(prev)


@pytest.mark.parametrize("name", sorted(POST_CASES))
def test_nms_port_matches_reference_nms(name):
    g = golden("post_" + name)
    heat, paf = POST_CASES[name](synth)
    assert _digest(heat, paf) == str(g["in_digest"]), "synthetic input drifted"
    jl = nms_port.joint_list_from_nms(nms_port.nms(heat, 0.1))
    ref = g["joint_list"]
    assert jl.shape == ref.shape
    if len(jl):
        np.testing.assert_array_equal(jl[:, [0, 1, 3, 4]], ref[:, [0, 1, 3, 4]])   # coordinates, ids, parts: exact
        assert np.abs(jl[:, 2] - ref[:, 2]).max() <= 5e-7                           # scores: IPP vs native cubic


@pytest.mark.parametrize("name", sorted(POST_CASES))
def test_pafprocess_port_matches_reference(name, built):
    g = golden("post_" + name)
    heat, paf = POST_CASES[name](synth)
    port = pafprocess_oracle.load_port()
    _, humans = glue_port.paf_to_pose(heat, paf, port)
    assert_humans_equal(humans, humans_rows_to_dicts(g["humans"]), score_tol=1e-6)
    if pafprocess_oracle.have_ref():      # the reference's own translation unit, same peaks -> bit-identical
        _, href = glue_port.paf_to_pose(heat, paf, pafprocess_oracle.load_ref())
        assert humans == href


def test_pafprocess_port_ties_and_scale(built):
    """Large crowded scenes produce exactly-equal candidate scores; std::sort's order is reproduced (against what the
    reference's own pafprocess.cpp made of the same scenes, tests/golden/make_golden.py)."""
    port, g = pafprocess_oracle.load_port(), golden("pafprocess_fuzz")
    for persons, seed in [(30, 31), (50, 5), (80, 7)]:
        heat, paf, _ = synth.stick_figures(persons, seed)
        a = glue_port.paf_to_pose(heat, paf, port)[1]
        b = humans_rows_to_dicts(g["crowd_%d_%d" % (persons, seed)])
        assert a == b and len(a) > persons // 2


def test_swig_typemap_errors(built):
    port = pafprocess_oracle.load_port()
    with pytest.raises(TypeError):
        port.process_paf(np.zeros((1, 1, 5), np.float64), np.zeros((8, 8, 19), np.float32), np.zeros((8, 8, 38), np.float32))


def test_cubic_resize_restatement_vs_opencv():
    """oracle/glue_port.resize_cubic (the composition oracle of the multi-scale averaging) against cv2.resize
    INTER_CUBIC: within 3e-7 of OpenCV's own code path (IPP off; cv2 evaluates the last row_length % 4 elements of a row
    in another order), identity for equal sizes, exact when the row length is a multiple of 4."""
    import cv2
    rs = np.random.RandomState(12)
    prev = cv2.ipp.useIPP()
    cv2.ipp.setUseIPP(False)
    try:
        for (h, w, dh, dw, c) in ((23, 23, 46, 46, 19), (69, 69, 46, 46, 38), (92, 92, 46, 46, 19), (6, 9, 12, 16, 38),
                                  (24, 33, 12, 16, 19), (46, 53, 46, 53, 19), (20, 30, 33, 47, 1)):
            src = rs.randn(h, w, c).astype(np.float32)
            ref = cv2.resize(src, (dw, dh), interpolation=cv2.INTER_CUBIC).reshape(dh, dw, c)
            mine = glue_port.resize_cubic(src, dh, dw)
            assert np.abs(mine - ref).max() <= 3e-7
            if (dw * c) % 4 == 0 or (h, w) == (dh, dw):
                np.testing.assert_array_equal(mine, ref)
    finally:
        cv2.ipp.setUseIPP(prev)
    x = rs.randn(46, 46, 19).astype(np.float32)
    np.testing.assert_array_equal(glue_port.resize_cubic(x, 46, 46), x)
    h1, p1 = rs.randn(12, 16, 19).astype(np.float32), rs.randn(12, 16, 38).astype(np.float32)
    ah, ap = glue_port.multi_scale_maps([(h1, p1)] * 4, (12, 16))
    np.testing.assert_array_equal(ah, h1)          # (4 x) / 4 is exact
    np.testing.assert_array_equal(ap, p1)


def _emulate_tc(x, w, b, ks, relu, pool, x_lo=None, w_lo=None, chunk=False, skip=None, shift=None, bias_roll=0):
    """The tensor-core kernel's fp32 arithmetic restated in numpy: per 64-channel block, tap-major, each k16 step adds
    its exact 16-product partial to the fp32 accumulator with one rounding; bf16x3 runs the terms A_hi W_hi, A_hi W_lo,
    A_lo W_hi per block, K-chunked (7x7: one chunk per filter row; otherwise one per block and term), chunks summed in
    fp32.  x: NHWC float32 bf16 values, w: OIHW float64 bf16 values.  Returns v = fp32(acc + bias), NCHW float64.
    Mutations: skip = (block, tap, k16) left out; shift = tap whose window is read one pixel to the right;
    bias_roll = bias of a neighbouring channel."""
    n, H, W, C = x.shape
    p = ks // 2
    planes = [np.pad(x.astype(np.float64), ((0, 0), (p, p), (p, p + 1), (0, 0)))]
    if x_lo is not None:
        planes.append(np.pad(x_lo.astype(np.float64), ((0, 0), (p, p), (p, p + 1), (0, 0))))
    terms = [(0, w)] if x_lo is None else [(0, w), (0, w_lo), (1, w)]
    O = w.shape[0]
    acc = np.zeros((n * H * W, O), np.float32)
    total = np.zeros_like(acc)
    for cb in range(C // 64):
        for pl, wt in terms:
            for tap in range(ks * ks):
                dy, dx = divmod(tap, ks)
                if chunk and ((ks == 7 and dx == 0) or (ks != 7 and tap == 0)):
                    acc[:] = 0
                ox = dx + (1 if shift == tap else 0)
                a = planes[pl][:, dy:dy + H, ox:ox + W, :].reshape(-1, C)
                for k in range(4):
                    if skip == (cb, tap, k):
                        continue
                    c0 = cb * 64 + 16 * k
                    part = a[:, c0:c0 + 16] @ wt[:, c0:c0 + 16, dy, dx].T
                    acc = (acc.astype(np.float64) + part).astype(np.float32)
                if chunk and ((ks == 7 and dx == ks - 1) or (ks != 7 and tap == ks * ks - 1)):
                    total = total + acc          # float32 + float32: round to nearest
    if not chunk:
        total = acc
    v = total + np.roll(b, -bias_roll).astype(np.float32)[None, :]
    return torch.from_numpy(v.reshape(n, H, W, O).transpose(0, 3, 1, 2).astype(np.float64))


def _layer(kind, seed):
    """A realistic layer: (x NHWC float32 bf16 values, x_lo, w OIHW fp32, b, ks, relu, pool, logical input channels).
    mconv1: a stage >= 2 Mconv1 of two groups reading the 192-channel concat buffer [PAF 0..37 | 0 0 | heat 40..58 |
    0 x 5 | features 64..191]; trunk: a 3x3 256 -> 256 layer with the fused 2x2 pool at width 92 (a partial last tile)."""
    from oracle import conv_check
    rs = np.random.RandomState(seed)
    if kind == "mconv1":
        n, H, W, C, cin, cout, ks, pool = 1, 16, 20, 192, 185, 256, 7, 0
        phys = np.r_[0:38, 40:59, 64:192]
    else:
        n, H, W, C, cin, cout, ks, pool = 1, 16, 92, 256, 256, 256, 3, 1
        phys = np.arange(256)
    full = np.zeros((n, H, W, C), np.float32)
    full[..., phys] = np.maximum(rs.randn(n, H, W, len(phys)), 0).astype(np.float32) * 1.5
    x = conv_check.bf16_round(torch.from_numpy(full.astype(np.float64))).numpy().astype(np.float32)
    x_lo = conv_check.bf16_round(torch.from_numpy(full.astype(np.float64) - x)).numpy().astype(np.float32)
    w = (rs.randn(cout, cin, ks, ks) * np.sqrt(2.0 / (cin * ks * ks))).astype(np.float32)
    b = (rs.rand(cout) * 0.2 - 0.1).astype(np.float32)
    return x, x_lo, w, b, ks, 1, pool, phys


def _check(x, x_lo, w, b, ks, relu, pool, phys, got_hi, got_lo=None):
    """The oracle's verdict for a layer (groups sharing the input are one conv here): Verdict of every output."""
    from oracle import conv_check
    C = x.shape[3]
    w_hi, w_lo = conv_check.split_weights(w)
    wp_hi = torch.zeros((w.shape[0], C, ks, ks), dtype=torch.float64)     # weights on the physical input channels
    wp_lo = torch.zeros_like(wp_hi)
    wp_hi[:, torch.from_numpy(phys)] = w_hi
    wp_lo[:, torch.from_numpy(phys)] = w_lo
    xt = torch.from_numpy(x.astype(np.float64)).permute(0, 3, 1, 2)
    bt = torch.from_numpy(b.astype(np.float64))
    split = got_lo is not None
    if split:
        r, S = conv_check.reference(xt, wp_hi, bt, ks, torch.from_numpy(x_lo.astype(np.float64)).permute(0, 3, 1, 2), wp_lo)
    else:
        r, S = conv_check.reference(xt, wp_hi, bt, ks)
    e = conv_check.U * conv_check.bound_coef(ks, C, split=split, chunk=split) * S
    if split:
        return conv_check.check_split(got_hi, got_lo, r, e, relu, pool)
    return conv_check.check_bf16(got_hi, r, e, relu, pool)


@pytest.mark.parametrize("kind", ["mconv1", "trunk"])
def test_conv_checker_accepts_the_kernel_arithmetic_and_rejects_each_mutation(kind):
    """oracle/conv_check.py is what the GPU layer test trusts, so it must be able to fail.  The kernel's own fp32
    accumulation order, emulated here, must pass; each of the faults a wgmma conv is prone to, applied to that emulation,
    must be caught by the 2^-22 bound at the real K (mconv1: K = 49 x 192 = 9 408; trunk: 9 x 256 = 2 304)."""
    from oracle import conv_check
    x, x_lo, w, b, ks, relu, pool, phys = _layer(kind, 7)
    w_hi, w_lo = conv_check.split_weights(w)
    wp_hi = np.zeros((w.shape[0], x.shape[3], ks, ks))
    wp_lo = np.zeros_like(wp_hi)
    wp_hi[:, phys], wp_lo[:, phys] = w_hi.numpy(), w_lo.numpy()

    def out_bf16(v):
        return conv_check.bf16_round(conf(v))

    def conf(v):
        return conv_check.f_act(v, relu, pool)

    v = _emulate_tc(x, wp_hi, b, ks, relu, pool)
    ok = _check(x, x_lo, w, b, ks, relu, pool, phys, out_bf16(v))
    print("%s bf16: emulated kernel accepted, max |v - r| / e = %.3f" % (kind, ok.ratio))
    assert bool(ok.ok.all()), conv_check.describe(ok, out_bf16(v), kind, pool)

    mutants = {
        "k16 slice of one tap dropped": _emulate_tc(x, wp_hi, b, ks, relu, pool, skip=(1, ks * ks // 2 + 1, 2)),
        "one tap read one pixel off": _emulate_tc(x, wp_hi, b, ks, relu, pool, shift=ks * ks - 1),
        "neighbour's bias": _emulate_tc(x, wp_hi, b, ks, relu, pool, bias_roll=1),
    }
    last = v.clone()
    last[..., -1] = v[..., -2]                     # the partial last tile's last column stored from its neighbour
    mutants["last partial tile column wrong"] = last
    swapped = v.clone()
    swapped[:, [5, 6]] = v[:, [6, 5]]              # two channels of an n-tile swapped
    mutants["two channels of an n-tile swapped"] = swapped
    for name, mv in mutants.items():
        verdict = _check(x, x_lo, w, b, ks, relu, pool, phys, out_bf16(mv))
        assert not bool(verdict.ok.all()), "%s: mutation '%s' passed the checker" % (kind, name)
        print("%s bf16: '%s' rejected (%d bad elements)" % (kind, name, int((~verdict.ok).sum())))
    if pool:                                       # the 2x2 max taken over the wrong column pair
        verdict = _check(x, x_lo, w, b, ks, relu, pool, phys, out_bf16(torch.roll(v, -1, 3)))
        assert not bool(verdict.ok.all()), "%s: wrong pool neighbour passed the checker" % kind

    # bf16x3: the three-term, K-chunked emulation passes; without the A_lo W_hi term it must not
    for drop_lo, should_pass in ((False, True), (True, False)):
        xl = np.zeros_like(x_lo) if drop_lo else x_lo      # without: A_hi W_hi + A_hi W_lo only
        fv = conf(_emulate_tc(x, wp_hi, b, ks, relu, pool, x_lo=xl, w_lo=wp_lo, chunk=True))
        hi = conv_check.bf16_round(fv)
        lo = conv_check.bf16_round(fv - hi)
        verdict = _check(x, x_lo, w, b, ks, relu, pool, phys, hi, lo)
        assert bool(verdict.ok.all()) == should_pass, (kind, drop_lo, conv_check.describe(verdict, hi + lo, kind, pool))
        print("%s bf16x3%s: %s, max |v - r| / e = %.3f" % (kind, " without A_lo W_hi" if drop_lo else "",
                                                           "accepted" if should_pass else "rejected", verdict.ratio))
