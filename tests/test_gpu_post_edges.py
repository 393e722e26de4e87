"""GPU (-m gpu): the device post-processing (peaks_kernel, the limb kernels, assemble_kernel) on adversarial heat maps
(oracle/synth.EDGE_CASES: plateaus, ties, maxima at the threshold, edge spikes, twin maxima), at the map sizes where the
kernels switch paths or refuse, and at every capacity limit.  Peaks must equal the oracle's NMS bit for bit and
persons the oracle's pafprocess (and, for the golden cases, what the reference itself made of the same maps)."""
import numpy as np
import pytest
import torch

from conftest import assert_humans_equal, golden, humans_rows_to_dicts, pkg_module
from oracle import glue_port, nms_port, pafprocess_oracle, synth

pytestmark = pytest.mark.gpu

THRESH = 0.1
CASES = {synth.edge_case_name(*c): c for c in synth.EDGE_CASES}
LIMB_PARTS, LIMB_PAF_CH = synth.LIMB_PARTS, synth.LIMB_PAF_CH


@pytest.fixture(scope="module")
def eng(built):
    return pkg_module("engine")


@pytest.fixture(scope="module")
def post1(eng):
    return eng.NativePost(0, batch_cap=1, peak_cap=2048, human_cap=2048)


def _oracle(heat, paf, thresh=THRESH):
    """(joint list, persons) of the oracle: nms_port + the C port of pafprocess.cpp."""
    return glue_port.paf_to_pose(heat, paf, pafprocess_oracle.load_port(), thresh=thresh)


def _run(post, heats, pafs, layout=1, thresh=THRESH):
    """Host maps [n, h, w, C] through post_run in `layout` (0 = [n, C, h, w])."""
    heats, pafs = np.stack(heats), np.stack(pafs)
    n, h, w = heats.shape[:3]
    if layout == 0:
        heats, pafs = heats.transpose(0, 3, 1, 2), pafs.transpose(0, 3, 1, 2)
    heats, pafs = np.ascontiguousarray(heats, np.float32), np.ascontiguousarray(pafs, np.float32)
    post.run(heats.ctypes.data, pafs.ctypes.data, False, layout, n, h, w, thresh)
    post.sync()


def _check_image(eng, post, i, heat, paf, thresh=THRESH, want=None):
    h, w = heat.shape[:2]
    jl, humans = want if want is not None else _oracle(heat, paf, thresh)
    assert post.status(i) == 0
    np.testing.assert_array_equal(post.peaks(i), jl)
    assert_humans_equal(eng.humans_to_dicts(post.humans(i), w * 8, h * 8), humans, score_tol=0.0)
    return jl, humans


# ------------------------------------------------------------------------------------------------ golden scenarios
@pytest.fixture(scope="module")
def edge(eng):
    """name -> (heat, paf, oracle joint list, oracle persons); the oracle is checked against the golden fixture here."""
    g = golden("post_edges")
    out = {}
    for name, c in CASES.items():
        heat, paf = synth.edge_maps(*c)
        jl, humans = _oracle(heat, paf)
        np.testing.assert_array_equal(jl, g[name + "_joint_list"])
        assert_humans_equal(humans, humans_rows_to_dicts(g[name + "_humans"]), score_tol=0.0)
        out[name] = (heat, paf, jl, humans)
    return out


@pytest.mark.parametrize("name", list(CASES))
def test_edge_scenario_layout1_from_host(name, eng, post1, edge):
    heat, paf, jl, humans = edge[name]
    _run(post1, [heat], [paf])
    _check_image(eng, post1, 0, heat, paf, want=(jl, humans))


def test_edge_scenarios_layout0_batches_per_shape(eng, edge):
    """Every golden scenario again as part of an NCHW batch of its shape: per-image results, no cross-talk."""
    shapes = {}
    for name, c in CASES.items():
        shapes.setdefault((c[2], c[3]), []).append(name)
    post = eng.NativePost(0, batch_cap=6, peak_cap=2048, human_cap=2048)
    for (h, w), names in sorted(shapes.items()):
        names = names + names[:1]          # a repeated image: the same results twice
        _run(post, [edge[n][0] for n in names], [edge[n][1] for n in names], layout=0)
        for i, n in enumerate(names):
            _check_image(eng, post, i, edge[n][0], edge[n][1], want=edge[n][2:])
        print((h, w), names)


def test_edge_scenarios_on_device_tensors(eng, edge):
    """on_device=1: torch tensors on the GPU, layout 1, the 46x46 scenarios as one batch."""
    names = [n for n, c in CASES.items() if (c[2], c[3]) == (46, 46)]
    heat = torch.from_numpy(np.stack([edge[n][0] for n in names])).cuda().contiguous()
    paf = torch.from_numpy(np.stack([edge[n][1] for n in names])).cuda().contiguous()
    post = eng.NativePost(0, batch_cap=len(names), peak_cap=2048, human_cap=2048)
    torch.cuda.synchronize()
    post.run(heat.data_ptr(), paf.data_ptr(), True, 1, len(names), 46, 46, THRESH,
             torch.cuda.current_stream().cuda_stream)
    post.sync()
    for i, n in enumerate(names):
        _check_image(eng, post, i, edge[n][0], edge[n][1], want=edge[n][2:])


@pytest.mark.parametrize("thresh", [0.05, 0.1, 0.3])
def test_thresholds(thresh, eng, post1):
    """Other thresholds on tie-heavy scenarios, and maxima exactly at / one float above float32(thresh)."""
    scen = [synth.edge_maps("plateau", 5, 46, 46), synth.edge_maps("quantised", 15, 46, 46),
            synth.edge_maps("twins", 53, 46, 46), synth.edge_maps("threshold", 61, 46, 46, thresh=thresh),
            synth.edge_maps("threshold", 62, 23, 31, thresh=thresh)]
    for k, (heat, paf) in enumerate(scen):
        _run(post1, [heat], [paf], thresh=thresh)
        jl, _ = _check_image(eng, post1, 0, heat, paf, thresh=thresh)
        if k >= 3:          # every pixel at float32(thresh) is no peak, and every maximum one float above is one
            above = np.nextafter(np.float32(thresh), np.float32(np.inf))
            want = sum(int((heat[:, :, p] == above).sum()) for p in range(18))
            assert len(jl) == want > 0


# ------------------------------------------------------------------------------------------------ map sizes
def _crowd(h, w, persons, seed):
    heat, paf, _ = synth.stick_figures(persons, seed, h=h, w=w)
    return heat, paf


@pytest.mark.parametrize("h,w,layouts", [(96, 128, (1, 0)), (97, 127, (1, 0)), (46, 276, (1,)), (92, 164, (1,)),
                                         (160, 310, (1,))])
def test_map_size_boundaries(h, w, layouts, eng, post1):
    """96x128 = 12 288 px: the limb scorer stages both PAF planes in shared memory; 97x127 and larger read them from
    global memory.  160x310 = 49 600 px is the largest plane the peaks kernel takes (200 KiB of shared memory)."""
    heat, paf = _crowd(h, w, 14, h * 1000 + w)
    edge_heat, _ = synth.edge_maps("border", h + w, h, w)
    heat[:, :, 4] = edge_heat[:, :, 4]          # spikes on every edge row and column in one part
    jl, humans = _oracle(heat, paf)
    assert len(humans) >= 5
    for layout in layouts:
        _run(post1, [heat], [paf], layout=layout)
        _check_image(eng, post1, 0, heat, paf, want=(jl, humans))
    print(h, w, "peaks", len(jl), "persons", len(humans))


def test_map_above_the_peaks_kernel_limit_is_refused(eng, post1):
    nat = pkg_module("_native")
    heat = np.zeros((160, 311, 19), np.float32)
    paf = np.zeros((160, 311, 38), np.float32)
    with pytest.raises(nat.B200PoseError):
        _run(post1, [heat], [paf])
    heat, paf = _crowd(46, 46, 5, 7)
    _run(post1, [heat], [paf])
    _check_image(eng, post1, 0, heat, paf)


# ------------------------------------------------------------------------------------------------ status bits
def _checker(h, w, n, parity=0, v=0.5):
    """A plane with exactly n isolated peaks of one value: the first n squares of a checkerboard, raster order."""
    ys, xs = np.mgrid[0:h, 0:w]
    on = ((ys + xs + parity) % 2 == 0).reshape(-1)
    idx = np.nonzero(on)[0][:n]
    m = np.zeros(h * w, np.float32)
    m[idx] = v
    return m.reshape(h, w)


def _expected_bits(jl, peak_cap, human_cap=None, humans=None, rows=None):
    """Status bits from the oracle's per-part peak counts and the capacity formulas of the kernels."""
    counts = np.bincount(jl[:, 4].astype(int), minlength=18) if len(jl) else np.zeros(18, int)
    st = 0
    if (counts > peak_cap).any():
        st |= 1
    if rows is not None and rows > 4 * peak_cap:
        st |= 4
    if human_cap is not None and len(humans) > human_cap:
        st |= 8
    return st


def _status_row(eng, post, images, expect, check_clean=True):
    """Runs [clean, case, clean] as one batch; the clean neighbours must be unaffected."""
    nat = pkg_module("_native")
    heats, pafs = [im[0] for im in images], [im[1] for im in images]
    _run(post, heats, pafs)
    for i, (heat, paf) in enumerate(images):
        if i == 1:
            assert post.status(i) == expect, (post.status(i), expect)
        elif check_clean:
            _check_image(eng, post, i, heat, paf)
    if expect & 0xF:
        with pytest.raises(nat.B200PoseError):
            post.check_status(len(images))
    else:
        post.check_status(len(images))


@pytest.mark.parametrize("cap,h,w", [(64, 24, 24), (2048, 64, 65)])
def test_status_bit1_peaks_per_part(cap, h, w, eng):
    post = eng.NativePost(0, batch_cap=3, peak_cap=cap, human_cap=256)
    clean = [_crowd(h, w, 2, 300 + k) for k in range(2)]
    zero_paf = np.zeros((h, w, 38), np.float32)
    for n in (cap, cap + 1):
        heat = np.zeros((h, w, 19), np.float32)
        heat[:, :, 3] = _checker(h, w, n)
        jl, humans = _oracle(heat, zero_paf)
        assert np.bincount(jl[:, 4].astype(int), minlength=18)[3] == n
        expect = _expected_bits(jl, cap)
        assert expect == (0 if n == cap else 1)
        _status_row(eng, post, [clean[0], (heat, zero_paf), clean[1]], expect)
        if expect == 0:
            np.testing.assert_array_equal(post.peaks(1), jl)
    if cap == 2048:          # full checkerboards: 64x64 gives exactly 2048 peaks, 64x65 gives 2080
        for hh, ww, want in ((64, 64, 2048), (64, 65, 2080)):
            m = _checker(hh, ww, hh * ww)
            assert len(nms_port.find_peaks(THRESH, m)) == want
            heat = np.zeros((hh, ww, 19), np.float32)
            heat[:, :, 3] = m
            _run(post, [heat], [np.zeros((hh, ww, 38), np.float32)])
            assert post.status(0) == (0 if want <= cap else 1)


def _field(h, w, limbs, segments):
    """PAF maps with unit direction (1, 0) on `limbs` only, in the low-res cells listed in `segments` [(y, x0, x1)]."""
    paf = np.zeros((h, w, 38), np.float32)
    for l in limbs:
        cx = LIMB_PAF_CH[l][0]
        for y, x0, x1 in segments:
            paf[y, x0:x1 + 1, cx] = 1.0
    return paf


def _pool_bits(jls, peak_cap, half):
    """Bit 2 per image of a batch, as limb_plan_kernel sets it: the candidate regions (na x nb + 2 entries per limb whose
    two parts both have peaks) of all images are laid out in (image, limb) order in ONE half-pool of `half` entries; a
    limb whose region ends past it is dropped and flags its image."""
    end, out = 0, []
    for jl in jls:
        c = np.minimum(np.bincount(jl[:, 4].astype(int), minlength=18) if len(jl) else np.zeros(18, int), peak_cap)
        st = 0
        for a, b in LIMB_PARTS:
            if c[a] > 0 and c[b] > 0:
                end += int(c[a]) * int(c[b]) + 2
                if end > half:
                    st |= 2
        out.append(st)
    return out


def _pool_scene(counts, h=64, w=64):
    """Checkerboard peaks: counts = {part: n}; a swirl on the PAF channels of every limb, so candidate scores vary."""
    heat = np.zeros((h, w, 19), np.float32)
    for k, (part, n) in enumerate(sorted(counts.items())):
        heat[:, :, part] = _checker(h, w, n, k % 2, np.float32(0.5 + 0.1 * k))
    ys, xs = np.mgrid[0:h, 0:w]
    paf = np.zeros((h, w, 38), np.float32)
    for l in range(len(LIMB_PARTS)):
        paf[:, :, LIMB_PAF_CH[l][0]] = np.cos(0.05 * ys + 0.3 * l).astype(np.float32)
        paf[:, :, LIMB_PAF_CH[l][1]] = np.sin(0.05 * xs + 0.3 * l).astype(np.float32)
    return heat, paf


def test_status_bit2_candidate_pool(eng):
    """batch_cap 1: the candidate half-pool holds 8 Mi keys.
    * Parts 1, 2 and 5 with 2048 peaks each make limbs 1-2 and 1-5 need 2 x (2048^2 + 2) > 8 Mi entries (bit 2); with
      2047 peaks in part 5 they fit.
    * Parts 1 and 2 with 2048 peaks, part 5 with 1983 and part 3 with 64 need 2048^2 + 2048 x 2047 + 6 <= 8 Mi entries:
      the two largest sorts and matchings the product path can meet (4 Mi and 4 Mi - 130 Ki candidate pairs) plus limb
      2-3.  Rows then hold parts 1, 2, 5 and 3, so persons are kept, and they expose which peaks the three matchings
      paired: they must equal the oracle's.  One more peak in part 5 sets bit 2."""
    nat = pkg_module("_native")
    post = eng.NativePost(0, batch_cap=1, peak_cap=2048, human_cap=256)
    half = (16 << 20) // 2
    for counts, full, persons in (({1: 2048, 2: 2048, 5: 2048}, True, False), ({1: 2048, 2: 2048, 5: 2047}, False, False),
                                  ({1: 2048, 2: 2048, 5: 1984, 3: 64}, True, False),
                                  ({1: 2048, 2: 2048, 5: 1983, 3: 64}, False, True)):
        heat, paf = _pool_scene(counts)
        jl = nms_port.joint_list_from_nms(nms_port.nms(heat, THRESH))
        expect = _pool_bits([jl], 2048, half)[0]
        assert expect == (2 if full else 0), counts
        _run(post, [heat], [paf])
        assert post.status(0) == expect, counts
        np.testing.assert_array_equal(post.peaks(0), jl)
        if expect:
            with pytest.raises(nat.B200PoseError):
                post.check_status(1)
            continue
        post.check_status(1)
        if persons:
            want = _oracle(heat, paf)
            assert len(want[1]) >= 20
            _check_image(eng, post, 0, heat, paf, want=want)
            print("largest sorts: %d persons identical to the oracle" % len(want[1]))


def test_status_bit2_is_shared_by_the_batch(eng):
    """batch_cap 3 ([clean, case, clean], 24 Mi keys): the case image's six limbs of 2048 x 2048 pairs need 24 Mi + 12
    entries (regions are sized by peak counts; its PAF maps are zero, so no candidate passes and no other bit is set).
    The pool is one buffer for the batch, laid out in image order: the image before the case is unaffected
    (status 0, peaks and persons identical), the case image and every image after it whose regions start past the end
    are flagged (bit 2, `check_status` raises) - loud, never silently wrong.  A clean batch afterwards is correct."""
    nat = pkg_module("_native")
    post = eng.NativePost(0, batch_cap=3, peak_cap=2048, human_cap=256)
    half = 3 * (16 << 20) // 2
    clean = [_crowd(64, 64, 3, 500 + k) for k in range(2)]
    case = (_pool_scene({p: 2048 for p in (0, 1, 2, 3, 5, 8, 11)})[0], np.zeros((64, 64, 38), np.float32))
    images = [clean[0], case, clean[1]]
    jls = [nms_port.joint_list_from_nms(nms_port.nms(im[0], THRESH)) for im in images]
    expect = _pool_bits(jls, 2048, half)
    assert expect == [0, 2, 2]
    _run(post, [im[0] for im in images], [im[1] for im in images])
    assert [post.status(i) for i in range(3)] == expect
    for i in range(3):
        np.testing.assert_array_equal(post.peaks(i), jls[i])
    _check_image(eng, post, 0, *clean[0])
    with pytest.raises(nat.B200PoseError):
        post.check_status(3)
    _run(post, [clean[0][0], clean[1][0], clean[0][0]], [clean[0][1], clean[1][1], clean[0][1]])
    for i, im in enumerate((clean[0], clean[1], clean[0])):
        _check_image(eng, post, i, *im)
    post.check_status(3)


def _disjoint_limbs_scene(h, w, n):
    """n peaks in both parts of each of seven limbs that share no part, each A peak joined to its own B peak two cells
    to the right by a field segment: 7 n rows of two parts, nothing kept."""
    limbs = [LIMB_PARTS.index(p) for p in ((1, 5), (2, 3), (6, 7), (8, 9), (11, 12), (0, 14), (15, 17))]
    heat = np.zeros((h, w, 19), np.float32)
    segs = []
    k = 0
    for y in range(1, h - 1, 6):
        for x in range(1, w - 3, 6):
            if k < n:
                segs.append((y, x, x + 2))
                k += 1
    assert k == n
    for l in limbs:
        a, b = LIMB_PARTS[l]
        for y, x0, x1 in segs:
            heat[y, x0, a] = 0.6
            heat[y, x1, b] = 0.7
    return heat, _field(h, w, limbs, segs), 7 * n


def _crowd_kept(h, w):
    heat, paf = _crowd(h, w, 30, 30)
    return heat, paf, _oracle(heat, paf)


def test_status_bits_each_on_its_own_image_and_the_sticky_accumulator(eng):
    """Bit 1 (peaks), 4 (rows) and 8 (persons), each on the middle image of [clean, case, clean]; status_accum(reset=True)
    returns their OR, and a clean run afterwards reports 0 everywhere."""
    h = w = 48
    crowd_heat, crowd_paf, (crowd_jl, crowd_humans) = _crowd_kept(h, w)
    k = len(crowd_humans)
    assert k >= 10
    cap = 64
    post = eng.NativePost(0, batch_cap=3, peak_cap=cap, human_cap=k - 1)
    clean = [_crowd(h, w, 1, 400 + i) for i in range(2)]
    post.status_accum(reset=True)
    acc = 0
    # bit 1
    heat = np.zeros((h, w, 19), np.float32)
    heat[:, :, 7] = _checker(h, w, cap + 1)
    zero = np.zeros((h, w, 38), np.float32)
    e1 = _expected_bits(nms_port.joint_list_from_nms(nms_port.nms(heat, THRESH)), cap)
    _status_row(eng, post, [clean[0], (heat, zero), clean[1]], e1)
    acc |= e1
    # bit 4: 7 x 64 = 448 rows > row_cap = 4 x 64; 7 x 36 = 252 fit
    for n in (cap, 36):
        heat, paf, rows = _disjoint_limbs_scene(h, w, n)
        jl, humans = _oracle(heat, paf)
        e4 = _expected_bits(jl, cap, rows=rows)
        assert e4 == (4 if n == cap else 0)
        _status_row(eng, post, [clean[0], (heat, paf), clean[1]], e4)
        if not e4:          # peaks only: every row holds two parts, so neither side keeps a person
            assert humans == [] and len(post.humans(1)) == 0
            np.testing.assert_array_equal(post.peaks(1), jl)
        acc |= e4
    # bit 8: k kept persons, human_cap k - 1
    e8 = _expected_bits(crowd_jl, cap, human_cap=k - 1, humans=crowd_humans)
    assert e8 == 8
    _status_row(eng, post, [clean[0], (crowd_heat, crowd_paf), clean[1]], e8)
    acc |= e8
    assert acc == 1 | 4 | 8
    assert post.status_accum(reset=True) == acc
    _run(post, [clean[0][0], clean[1][0], clean[0][0]], [clean[0][1], clean[1][1], clean[0][1]])
    assert [post.status(i) for i in range(3)] == [0, 0, 0]
    assert post.status_accum() == 0


def test_status_bit8_boundary(eng):
    """human_cap = k keeps all k persons of a crowd (status 0, identical persons); k - 1 sets bit 8."""
    h = w = 48
    heat, paf, (jl, humans) = _crowd_kept(h, w)
    k = len(humans)
    for cap, expect in ((k, 0), (k - 1, 8)):
        post = eng.NativePost(0, batch_cap=1, peak_cap=64, human_cap=cap)
        assert _expected_bits(jl, 64, human_cap=cap, humans=humans) == expect
        _run(post, [heat], [paf])
        assert post.status(0) == expect
        if expect == 0:
            _check_image(eng, post, 0, heat, paf, want=(jl, humans))
