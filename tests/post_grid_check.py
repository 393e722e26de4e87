"""Shared by tests/test_post_grid_host.py and tests/test_gpu_post_grid.py: the scenarios on which the PAF scoring and
range sorting kernels are checked at every grid size, and the scoring work queue they make.

limb_score_kernel takes work items from a global cursor, four at a time: an item is 2048 consecutive (a, b) pairs of
one (image, limb), and the items of all (image, limb) are laid out in (image, limb) order (limb_plan_kernel).  A block
stages the two PAF planes of an item's (image, limb) and keeps them while the following items belong to it.  The
scenarios below are built from peak counts so that this queue has the shapes that matter: a group of four items that
spans two images' lists of the same limb, groups that cross a limb and an image boundary, and more groups than blocks
at every grid size."""
import numpy as np

from conftest import POST_CASES
from oracle import nms_port, synth

CHUNK_PAIRS = 2048          # pairs per scoring work item (kLimbChunkPairs)
GROUP = 4                   # work items per grab of the cursor
H100_SMS = 132
LIMB_PARTS, LIMB_PAF_CH = synth.LIMB_PARTS, synth.LIMB_PAF_CH
THRESH = 0.1

# same-limb batch: only parts 1 and 2 have peaks, so limb 0 (li = 0 and li = 19) is the only one with pairs; 70 x 70
# and 60 x 90 pairs are 3 items each, so the first group holds li 0's three items and li 19's first
SAME_LIMB_COUNTS = ({1: 70, 2: 70}, {1: 60, 2: 90})
# boundary batch: item counts 3, 2, 1 | 2, 2, 3 | 2, 2, 1 per (image, limb), none a multiple of four
CROSSING_COUNTS = ({1: 90, 2: 50, 5: 33, 6: 41}, {1: 45, 2: 70, 3: 61, 5: 80}, {0: 50, 1: 77, 14: 66, 16: 20})
NOISE_SEEDS = range(5)      # five 7 000-peak noise maps: more groups than 12 x 132 blocks
# the status-bit-2 boundary scene of tests/test_gpu_post_edges.py: 4 Mi + 4 Mi - 130 Ki candidate pairs
BIT2_COUNTS = {1: 2048, 2: 2048, 5: 1983, 3: 64}


def joint_list(heat):
    return nms_port.joint_list_from_nms(nms_port.nms(heat, THRESH, 18))


def part_counts(heat):
    jl = joint_list(heat)
    return np.bincount(jl[:, 4].astype(int), minlength=18) if len(jl) else np.zeros(18, int)


def spaced_scene(counts, seed, h, w):
    """(heat, paf) HWC float32: counts = {part: n} isolated peaks per part on cells (even y, even x) - no two of a part
    touch, so each is a peak of its own - with random values; every limb's PAF field is a smooth swirl whose phase
    depends on `seed`, so two scenes of one peak layout score their pairs differently."""
    rs = np.random.RandomState(seed)
    cells = [(y, x) for y in range(0, h, 2) for x in range(0, w, 2)]
    heat = np.zeros((h, w, 19), np.float32)
    for part, n in sorted(counts.items()):
        for k in rs.choice(len(cells), n, replace=False):
            y, x = cells[k]
            heat[y, x, part] = np.float32(rs.uniform(0.3, 0.95))
    ys, xs = np.mgrid[0:h, 0:w]
    paf = np.zeros((h, w, 38), np.float32)
    ph = rs.uniform(0, 2 * np.pi, (len(LIMB_PARTS), 2))
    for l, (cx, cy) in enumerate(LIMB_PAF_CH):
        paf[:, :, cx] = np.cos(0.11 * ys + 0.07 * xs + ph[l, 0])
        paf[:, :, cy] = np.sin(0.05 * ys - 0.13 * xs + ph[l, 1])
    return heat, paf


def scenarios():
    """name -> (list of (heat, paf) HWC images, layout, post-processing settings name or None).  Each is one batch."""
    out = {}
    stick = {k: POST_CASES[k](synth) for k in ("p1", "p3", "p8", "p30", "noise0", "p5_40x52")}
    out["golden46"] = ([stick[k] for k in ("p1", "p3", "p8", "p30", "noise0")], 1, None)
    out["golden40x52"] = ([stick["p5_40x52"]], 1, None)
    edges = {synth.edge_case_name(*c): c for c in synth.EDGE_CASES}
    for hw in ("46x46", "23x31"):
        names = [n for n in edges if n.endswith(hw) and n.split("_")[0] in ("plateau", "twins")]
        out["edges" + hw] = ([synth.edge_maps(*edges[n]) for n in names], 0, None)
    for h, w in ((46, 46), (97, 127)):
        for layout in (0, 1):
            tag = "%dx%d_l%d" % (h, w, layout)
            out["samelimb" + tag] = ([spaced_scene(c, 10 + i, h, w) for i, c in enumerate(SAME_LIMB_COUNTS)], layout,
                                     None)
            out["crossing" + tag] = ([spaced_scene(c, 20 + i, h, w) for i, c in enumerate(CROSSING_COUNTS)], layout,
                                     None)
    out["loose46"] = (out["golden46"][0], 1, "loose")
    out["noise46"] = ([synth.noise_maps(s) for s in NOISE_SEEDS], 1, None)
    return out


def bit2_scene():
    """The 64 x 64 scene of BIT2_COUNTS: one value per part on a checkerboard, a swirl on every limb (as in
    tests/test_gpu_post_edges.py)."""
    h = w = 64
    ys, xs = np.mgrid[0:h, 0:w]
    heat = np.zeros((h, w, 19), np.float32)
    for k, (part, n) in enumerate(sorted(BIT2_COUNTS.items())):
        on = ((ys + xs + k % 2) % 2 == 0).reshape(-1)
        m = np.zeros(h * w, np.float32)
        m[np.nonzero(on)[0][:n]] = np.float32(0.5 + 0.1 * k)
        heat[:, :, part] = m.reshape(h, w)
    paf = np.zeros((h, w, 38), np.float32)
    for l in range(len(LIMB_PARTS)):
        paf[:, :, LIMB_PAF_CH[l][0]] = np.cos(0.05 * ys + 0.3 * l).astype(np.float32)
        paf[:, :, LIMB_PAF_CH[l][1]] = np.sin(0.05 * xs + 0.3 * l).astype(np.float32)
    return heat, paf


def work_items(counts_per_image):
    """The scoring work queue of a batch: one entry per item, (image, limb) in item order.  counts_per_image: the
    18 peak counts of every image (pool capacity is not modelled: the scenarios stay far below it)."""
    items = []
    for img, c in enumerate(counts_per_image):
        for limb, (a, b) in enumerate(LIMB_PARTS):
            pairs = int(c[a]) * int(c[b])
            items += [(img, limb)] * (-(-pairs // CHUNK_PAIRS))
    return items


def groups(items):
    """The items of each grab of the cursor, in order."""
    return [items[g:g + GROUP] for g in range(0, len(items), GROUP)]


def sort_inputs():
    """The 162 key sets of tests/test_gpu.py's device sort test (high words; the low word is the index), in order."""
    rs = np.random.RandomState(0)
    out = []
    for n in [1, 2, 3, 15, 16, 17, 18, 31, 32, 33, 64, 65, 100, 257, 1000, 2048, 4095, 4096, 4097, 5000, 9000, 20000,
              70000, 300000]:
        for distinct in (1, 2, 7, max(1, n // 3), 1 << 30):
            out.append(rs.randint(0, distinct, size=n))
    for n in (17, 33, 100, 1000, 4096, 5000, 50000):
        for hi in (np.arange(n), np.arange(n)[::-1], np.minimum(np.arange(n), np.arange(n)[::-1]), np.arange(n) % 2,
                   np.arange(n) % 17, (np.arange(n) * 7919) % 1013):
            out.append(np.ascontiguousarray(hi))
    return out
