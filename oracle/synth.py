"""ORACLE-side synthetic input generators (test infrastructure only): seeded stick-figure heat/PAF maps in the
reference's 19-heat / 38-PAF COCO layout (SURVEY.md appendix B), and noise maps.  These are INPUTS for parity
tests, not a restatement of any reference function."""
import numpy as np

LIMB_PARTS = [(1, 2), (1, 5), (2, 3), (3, 4), (5, 6), (6, 7), (1, 8), (8, 9), (9, 10), (1, 11), (11, 12), (12, 13),
              (1, 0), (0, 14), (14, 16), (0, 15), (15, 17), (2, 16), (5, 17)]
LIMB_PAF_CH = [(12, 13), (20, 21), (14, 15), (16, 17), (22, 23), (24, 25), (0, 1), (2, 3), (4, 5), (6, 7), (8, 9),
               (10, 11), (28, 29), (30, 31), (34, 35), (32, 33), (36, 37), (18, 19), (26, 27)]
# canonical skeleton in a unit box (x, y), 18 COCO parts
_SKEL = np.array([[.50, .08], [.50, .22], [.36, .22], [.30, .40], [.27, .56], [.64, .22], [.70, .40], [.73, .56],
                  [.42, .55], [.41, .75], [.40, .95], [.58, .55], [.59, .75], [.60, .95], [.46, .05], [.54, .05],
                  [.41, .07], [.59, .07]])


def stick_figures(num_persons, seed, h=46, w=46, stride=8, sigma=7.0, paf_width=6.0, drop_prob=0.1):
    """Returns (heat [h,w,19] float32, paf [h,w,38] float32, keypoints [P,18,3] (x,y,visible) in image pixels)."""
    rs = np.random.RandomState(seed)
    H, W = h * stride, w * stride
    heat = np.zeros((h, w, 19), np.float32)
    paf = np.zeros((h, w, 38), np.float32)
    cnt = np.zeros((h, w, 19), np.float32)
    ys, xs = np.mgrid[0:h, 0:w]
    cx = xs * stride + stride / 2.0 - 0.5
    cy = ys * stride + stride / 2.0 - 0.5
    kps = np.zeros((num_persons, 18, 3))
    for p in range(num_persons):
        size = rs.uniform(0.28, 0.6) * min(H, W)
        ox = rs.uniform(0, W - size * 0.5)
        oy = rs.uniform(0, H - size)
        ang = rs.uniform(-0.35, 0.35)
        rot = np.array([[np.cos(ang), -np.sin(ang)], [np.sin(ang), np.cos(ang)]])
        pts = (_SKEL - 0.5) @ rot.T * size + [ox + size * 0.5, oy + size * 0.5] + rs.normal(0, size * 0.015, (18, 2))
        vis = (rs.rand(18) > drop_prob) & (pts[:, 0] >= 0) & (pts[:, 0] < W) & (pts[:, 1] >= 0) & (pts[:, 1] < H)
        kps[p, :, :2] = pts
        kps[p, :, 2] = vis
        for j in range(18):
            if not vis[j]:
                continue
            g = np.exp(-((cx - pts[j, 0]) ** 2 + (cy - pts[j, 1]) ** 2) / (2 * sigma * sigma))
            heat[:, :, j] = np.maximum(heat[:, :, j], g * rs.uniform(0.75, 1.0))
        for l, (a, b) in enumerate(LIMB_PARTS):
            if not (vis[a] and vis[b]):
                continue
            v = pts[b] - pts[a]
            n = np.linalg.norm(v)
            if n < 1e-3:
                continue
            u = v / n
            rx, ry = cx - pts[a, 0], cy - pts[a, 1]
            along = rx * u[0] + ry * u[1]
            perp = np.abs(rx * u[1] - ry * u[0])
            m = (along >= 0) & (along <= n) & (perp <= paf_width)
            paf[:, :, LIMB_PAF_CH[l][0]][m] += u[0]
            paf[:, :, LIMB_PAF_CH[l][1]][m] += u[1]
            cnt[:, :, l][m] += 1
    for l in range(19):
        m = cnt[:, :, l] > 1
        for ch in LIMB_PAF_CH[l]:
            paf[:, :, ch][m] /= cnt[:, :, l][m]
    heat[:, :, 18] = 1.0 - heat[:, :, :18].max(axis=2)
    heat += rs.normal(0, 0.004, heat.shape).astype(np.float32)   # breaks exact ties / plateaus
    paf += rs.normal(0, 0.004, paf.shape).astype(np.float32)
    return heat.astype(np.float32), paf.astype(np.float32), kps


def noise_maps(seed, h=46, w=46, heat_scale=0.45, paf_scale=0.6):
    """Maps with the statistics of a random-weight network (thousands of peaks): the stress case."""
    rs = np.random.RandomState(seed)
    heat = (rs.standard_normal((h, w, 19)) * heat_scale).astype(np.float32)
    paf = (rs.standard_normal((h, w, 38)) * paf_scale).astype(np.float32)
    return heat, paf


# ---------------------------------------------------------------------------------------------------------------
# Fuzz scenarios for the pafprocess stage (joint list + low-resolution PAF maps, no NMS involved): used to compare the
# reference's compiled pafprocess.cpp with the product's cores on inputs the stick-figure fixtures do not reach
# (cross links between persons, duplicated peaks on one pixel, exact score ties, masked fields).
_LIMBS = [(1, 2), (1, 5), (2, 3), (3, 4), (5, 6), (6, 7), (1, 8), (8, 9), (9, 10), (1, 11), (11, 12), (12, 13), (1, 0),
          (0, 14), (14, 16), (0, 15), (15, 17), (2, 16), (5, 17)]                       # pafprocess.h:21-24
_PAFCH = [(12, 13), (20, 21), (14, 15), (16, 17), (22, 23), (24, 25), (0, 1), (2, 3), (4, 5), (6, 7), (8, 9), (10, 11),
          (28, 29), (30, 31), (34, 35), (32, 33), (36, 37), (18, 19), (26, 27)]           # pafprocess.h:16-19


def fuzz_field(rs, h, w, kind):
    """Random peaks (kind: 'uniform' | 'cluster' | 'ties') + per-limb (nearly) constant direction fields."""
    maxp = int(rs.choice([1, 2, 3, 5, 8]))
    rows = []
    centers = rs.randint(8, min(h, w) * 8 - 8, (int(rs.randint(1, 6)), 2))
    for part in range(18):
        for _ in range(int(rs.randint(0, maxp + 1))):
            if kind in ("cluster", "ties") and rs.rand() < 0.8:
                c = centers[rs.randint(len(centers))]
                spread = 3 if kind == "ties" else 40
                x = int(np.clip(c[0] + rs.randint(-spread, spread + 1), 0, w * 8 - 1))
                y = int(np.clip(c[1] + rs.randint(-spread, spread + 1), 0, h * 8 - 1))
            else:
                x, y = int(rs.randint(0, w * 8)), int(rs.randint(0, h * 8))
            rows.append((x, y, float(np.float32(rs.choice([0.2, 0.5, 0.9, rs.rand()]))), 0, part))
    jl = np.array(rows, np.float32).reshape(-1, 5)
    jl[:, 3] = np.arange(len(jl))
    return jl, direction_fields(rs, h, w, kind == "ties")


def direction_fields(rs, h, w, ties):
    """PAF maps [h, w, 38] float32: per limb a constant direction and magnitude, with Gaussian noise (none when `ties`:
    the angles are then multiples of 90 degrees or 45 degrees, so many candidates score exactly alike), and in 30 % of
    the limbs a random mask that zeroes 30 % of the pixels."""
    paf = np.zeros((h, w, 38), np.float32)
    for ch in range(0, 38, 2):
        ang = rs.choice([0, np.pi / 2, np.pi, 3 * np.pi / 2, np.pi / 4]) if ties else rs.rand() * 2 * np.pi
        mag = rs.choice([0.3, 0.6, 1.0])
        noise = 0.0 if ties else 0.3
        paf[:, :, ch] = np.cos(ang) * mag + noise * rs.randn(h, w)
        paf[:, :, ch + 1] = np.sin(ang) * mag + noise * rs.randn(h, w)
        if rs.rand() < 0.3:
            paf[:, :, ch:ch + 2] *= (rs.rand(h, w, 1) < 0.7)
    return np.ascontiguousarray(paf.astype(np.float32))


def fuzz_persons(rs, h, w):
    """1-6 loosely person-shaped peak sets with their true limbs drawn into the PAF maps, random cross links between
    persons (ambiguous assignments, merges of partial persons) and duplicated peaks (exact score ties)."""
    K = int(rs.randint(1, 7))
    pts = {}
    for k in range(K):
        c = rs.randint(40, min(h, w) * 8 - 40, 2)
        sc = rs.randint(10, 45)
        for part in range(18):
            if rs.rand() < 0.85:
                pts[(k, part)] = (int(np.clip(c[0] + rs.randint(-sc, sc + 1), 0, w * 8 - 1)),
                                  int(np.clip(c[1] + rs.randint(-sc, sc + 1), 0, h * 8 - 1)))
    rows = []
    for part in range(18):
        for k in range(K):
            if (k, part) in pts:
                x, y = pts[(k, part)]
                rows.append((x, y, float(np.float32(rs.choice([0.3, 0.6, 0.95]))), 0, part))
                if rs.rand() < 0.15:
                    rows.append((x + int(rs.randint(0, 2)), y, float(np.float32(0.6)), 0, part))
    jl = np.array(rows, np.float32).reshape(-1, 5)
    jl[:, 3] = np.arange(len(jl))
    paf = np.zeros((h, w, 38), np.float32)

    def draw(a, b, chx, chy, mag):
        ax, ay, bx, by = a[0] / 8.0, a[1] / 8.0, b[0] / 8.0, b[1] / 8.0
        d = np.array([bx - ax, by - ay])
        nrm = np.linalg.norm(d)
        if nrm < 1e-6:
            return
        u = d / nrm
        for t in np.linspace(0, 1, int(nrm * 2) + 2):
            px, py = ax + t * d[0], ay + t * d[1]
            for ox in (-1, 0, 1):
                for oy in (-1, 0, 1):
                    xi, yi = int(round(px)) + ox, int(round(py)) + oy
                    if 0 <= xi < w and 0 <= yi < h:
                        paf[yi, xi, chx] = u[0] * mag
                        paf[yi, xi, chy] = u[1] * mag
    for l, (pa, pb) in enumerate(_LIMBS):
        for k in range(K):
            if (k, pa) in pts and (k, pb) in pts and rs.rand() < 0.9:
                draw(pts[(k, pa)], pts[(k, pb)], _PAFCH[l][0], _PAFCH[l][1], float(rs.choice([0.5, 0.8, 1.0])))
            k2 = int(rs.randint(K))
            if k2 != k and (k, pa) in pts and (k2, pb) in pts and rs.rand() < 0.35:
                draw(pts[(k, pa)], pts[(k2, pb)], _PAFCH[l][0], _PAFCH[l][1], float(rs.choice([0.5, 0.8, 1.0])))
    return jl, np.ascontiguousarray(paf)


# ---------------------------------------------------------------------------------------------------------------
# Adversarial heat maps for the peak stage: exact ties, plateaus, values exactly at the threshold, peaks on every
# edge row / column, coincident refinements.  Each plane generator returns one [h, w] float32 plane of part `part`.
_LEVELS = (0.35, 0.5, 0.8)     # plateau / spike values: above every threshold the tests use (0.05, 0.1, 0.3)


def _low(rs, h, w, thresh):
    """Background strictly below the threshold: its local maxima are never peaks."""
    return (rs.rand(h, w) * 0.5 * thresh).astype(np.float32)


def _plane_plateau(rs, h, w, thresh, part):
    """Equal-valued rectangles, a third of them on the map's edge, half of them with an equal-valued neighbour."""
    m = _low(rs, h, w, thresh)
    for _ in range(1 + h * w // 120):
        v = np.float32(rs.choice(_LEVELS))
        rh, rw = int(rs.randint(1, min(h, 5) + 1)), int(rs.randint(1, min(w, 5) + 1))
        y0 = int(rs.choice([0, h - rh])) if rs.rand() < 0.3 else int(rs.randint(0, h - rh + 1))
        x0 = int(rs.choice([0, w - rw])) if rs.rand() < 0.3 else int(rs.randint(0, w - rw + 1))
        m[y0:y0 + rh, x0:x0 + rw] = v
        if rs.rand() < 0.5:          # an equal plateau right of / below it
            if rs.rand() < 0.5:
                m[y0:y0 + max(1, rh - 1), x0 + rw:x0 + rw + 2] = v
            else:
                m[y0 + rh:y0 + rh + 2, x0:x0 + max(1, rw - 1)] = v
    return m


def _plane_quantised(rs, h, w, thresh, part):
    """Values on the grid k/16: smooth blobs rounded to it (wide plateaus, ties inside the up-sampled patch) or white
    noise on it (many equal neighbours)."""
    if rs.rand() < 0.3:
        return (rs.randint(0, 17, (h, w)) / 16.0).astype(np.float32)
    ys, xs = np.mgrid[0:h, 0:w]
    m = np.zeros((h, w))
    for _ in range(1 + h * w // 150):
        cy, cx, s = rs.uniform(-1, h), rs.uniform(-1, w), rs.uniform(1.0, 4.0)
        m = np.maximum(m, rs.uniform(0.3, 1.0) * np.exp(-((ys - cy) ** 2 + (xs - cx) ** 2) / (2 * s * s)))
    return (np.floor(m * 16 + 0.5) / 16).astype(np.float32)


def _plane_checkerboard(rs, h, w, thresh, part):
    """One value on every other pixel, zero on the rest: ceil or floor of h*w/2 peaks (exactly h*w/2 when h*w is
    even), all of one value."""
    ys, xs = np.mgrid[0:h, 0:w]
    return np.where((ys + xs + part) % 2 == 0, np.float32(rs.choice(_LEVELS)), np.float32(0)).astype(np.float32)


def _plane_threshold(rs, h, w, thresh, part):
    """Isolated local maxima exactly at float32(thresh) (not peaks: the test is `>`) and at the next float32 above it
    (peaks), alternating, on a grid of pitch 3."""
    m = _low(rs, h, w, thresh)
    at = np.float32(thresh)
    above = np.nextafter(at, np.float32(np.inf))
    k = int(rs.randint(2))
    for y in range(int(rs.randint(3)), h, 3):
        for x in range(int(rs.randint(3)), w, 3):
            m[y, x] = above if k % 2 else at
            k += 1
    return m


def _edge_lines(n):
    return sorted({i for i in (0, 1, 2, n - 3, n - 2, n - 1) if 0 <= i < n})


def _plane_border(rs, h, w, thresh, part):
    """Isolated spikes (with a lower random shoulder) on rows and columns 0, 1, 2, n-3, n-2, n-1 and in the four
    corners: both sides of the device's interior / border split (2 <= x <= w-3 and 2 <= y <= h-3)."""
    m = _low(rs, h, w, thresh)
    spots = [(0, 0), (0, w - 1), (h - 1, 0), (h - 1, w - 1)]
    spots += [(y, int(rs.randint(w))) for y in _edge_lines(h)]
    spots += [(int(rs.randint(h)), x) for x in _edge_lines(w)]
    for y, x in spots:
        v = np.float32(rs.uniform(0.2, 1.0))
        for dy, dx in ((-1, 0), (1, 0), (0, -1), (0, 1)):
            if 0 <= y + dy < h and 0 <= x + dx < w and m[y + dy, x + dx] < 0.2:
                m[y + dy, x + dx] = np.float32(v * rs.uniform(0.3, 0.9))
    for y, x in spots:       # spikes last, so a shoulder never covers one
        m[y, x] = max(m[y, x], np.float32(rs.uniform(0.2, 1.0)))
    return m


def _plane_twins(rs, h, w, thresh, part):
    """Pairs of adjacent equal maxima on a grid of pitch 5: both are peaks, and their x8 refinements read the same
    pixels with the same coefficients, so two peak ids usually refine to one up-sampled position."""
    m = _low(rs, h, w, thresh)
    for y in range(int(rs.randint(5)), h, 5):
        for x in range(int(rs.randint(5)), w, 5):
            v = np.float32(rs.choice(_LEVELS))
            m[y, x] = v
            if rs.rand() < 0.5 and x + 1 < w:
                m[y, x + 1] = v
            elif y + 1 < h:
                m[y + 1, x] = v
    return m


EDGE_KINDS = {"plateau": _plane_plateau, "quantised": _plane_quantised, "checkerboard": _plane_checkerboard,
              "threshold": _plane_threshold, "border": _plane_border, "twins": _plane_twins}


def edge_maps(kind, seed, h, w, thresh=0.1):
    """(heat [h, w, 19], paf [h, w, 38]) float32: every heat plane from the generator `kind`, PAF maps from
    `direction_fields` (exact ties in half of the seeds), so that duplicated and tied peaks reach scoring and matching."""
    rs = np.random.RandomState(seed)
    gen = EDGE_KINDS[kind]
    heat = np.stack([gen(rs, h, w, thresh, part) for part in range(19)], axis=2).astype(np.float32)
    paf = direction_fields(rs, h, w, bool(rs.rand() < 0.5))
    return np.ascontiguousarray(heat), paf


# (kind, seed, h, w) of the golden fixture tests/golden/post_edges.npz (reference NMS + pafprocess.cpp at thresh 0.1)
EDGE_CASES = (
    ("plateau", 1, 1, 1), ("plateau", 2, 3, 3), ("plateau", 3, 5, 5), ("plateau", 4, 23, 31), ("plateau", 5, 46, 46),
    ("quantised", 11, 1, 7), ("quantised", 12, 7, 1), ("quantised", 13, 4, 5), ("quantised", 14, 23, 31),
    ("quantised", 15, 46, 46),
    ("checkerboard", 21, 1, 7), ("checkerboard", 22, 4, 5), ("checkerboard", 23, 16, 16),
    ("threshold", 31, 3, 3), ("threshold", 32, 23, 31), ("threshold", 33, 46, 46),
    ("border", 41, 5, 5), ("border", 42, 7, 1), ("border", 43, 23, 31), ("border", 44, 46, 46), ("border", 45, 64, 64),
    ("twins", 51, 4, 5), ("twins", 52, 23, 31), ("twins", 53, 46, 46),
)


def edge_case_name(kind, seed, h, w):
    return "%s_%d_%dx%d" % (kind, seed, h, w)
