"""ORACLE (test infrastructure only).  The per-launch check of oracle/conv_check.py applied frame by frame to a launch of a
ragged batch (DESIGN.md §1.1), and to a uniform one as the case whose frames fill the canvas.

A ragged batch runs its frames on one canvas; the extents table holds each frame's padded size at the network input, and
a launch at 1/2^s of that resolution keeps ext >> s of it (add_plan's ext_shift, which counts the launch's own 2x2 pool
too).  For one image of one launch:

  * inside the frame's extent at the output resolution the stored values must lie in the interval the caller's verdict
    gives for a float64 convolution of the launch's own input planes cropped to the frame's extent at the input
    resolution: canvas pixels beyond the frame are +0 by the ragged rule, so a frame's edge sees zero padding, never a
    neighbour's pixels or stale data;
  * outside the extent every 16-bit word of every plane in the channels the launch writes, and every element of the fp32
    maps it writes, is +0 (bit pattern 0);
  * channels outside the launch's slice are bit-unchanged, and the pad channels of a head slice are 0.

Everything here takes host numpy arrays, so tests/test_ragged_check_host.py runs it on arrays it builds."""
import numpy as np

from oracle import conv_check


def ext_shift(h, H, pool=0):
    """add_plan's shift: the smallest s with h << s >= H (h: the launch's input height, H: the network input's), plus
    the launch's pool."""
    s = 0
    while (h << s) < H:
        s += 1
    return s + pool


def extents(ext, h, H, pool):
    """(input extent, output extent) of a frame whose padded size at the network input is ext = (He, We), for a launch
    whose input height is h on a network input of height H."""
    s_in = ext_shift(h, H)
    s_out = s_in + pool
    return (ext[0] >> s_in, ext[1] >> s_in), (ext[0] >> s_out, ext[1] >> s_out)


def check_image(verdicts, src, after, before, ext, h, H, pool, written, pad, maps=(), where=""):
    """One image of one launch.

    verdicts(src_in, got_in, maps_in) -> (list of (name, Verdict, got) per interval check, list of failure messages):
        the caller's interval checks on the frame's own region: src_in are the input planes cropped to the input extent
        (uint16 [hi, wi, C]), got_in the output planes cropped to the output extent, maps_in the fp32 maps cropped to it.
    src, after: lists of uint16 [h, w, C] planes of this image (bf16x3: hi and residual), before: the output planes as the
    launch found them, or None (nothing to compare); written: bool [C_out] the launch's channel slice; pad: the written
    channels beyond the conv's outputs (0 everywhere); maps: float32 [C, ho, wo] fp32 maps the launch writes.
    Returns (failure messages, worst |v - r| / e)."""
    (hi, wi), (ho, wo) = extents(ext, h, H, pool)
    vs, fails = verdicts([p[:hi, :wi] for p in src], [p[:ho, :wo] for p in after], [m[:, :ho, :wo] for m in maps])
    ratio = 0.0
    for name, v, got in vs:
        if not bool(v.ok.all()):
            fails.append(conv_check.describe(v, got, "%s %s" % (where, name), pool))
        ratio = max(ratio, v.ratio)
    fails += outside_fails(after, maps, ho, wo, written, where)
    for k, p in enumerate(after):
        if pad and np.any(p[..., pad]):
            fails.append("%s: pad channels %s (plane %d) are not +0" % (where, pad, k))
        if before is not None and not written.all() and not np.array_equal(p[..., ~written], before[k][..., ~written]):
            fails.append("%s: channels outside the launch's slice changed (plane %d)" % (where, k))
    return fails, ratio


def outside_fails(after, maps, ho, wo, written, where=""):
    """Every word of the written channels of the planes, and every fp32 map element, beyond [:ho, :wo] must be +0."""
    fails = []
    for k, p in enumerate(after):
        q = p[..., written]
        bad = int(np.count_nonzero(q[ho:])) + int(np.count_nonzero(q[:ho, wo:]))
        if bad:
            fails.append("%s: plane %d has %d non-zero words outside the frame's %dx%d extent" % (where, k, bad, ho, wo))
    for k, m in enumerate(maps):
        u = np.ascontiguousarray(m, np.float32).view(np.uint32)
        bad = int(np.count_nonzero(u[:, ho:])) + int(np.count_nonzero(u[:, :ho, wo:]))
        if bad:
            fails.append("%s: fp32 map %d has %d elements outside the frame's %dx%d extent that are not +0"
                         % (where, k, bad, ho, wo))
    return fails
