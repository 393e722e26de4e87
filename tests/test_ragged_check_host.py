"""CPU: the per-frame verdict of tests/ragged_check.py, as tests/test_gpu_conv_tc_matrix.py applies it, accepts a host
emulation of a ragged conv_tc_kernel launch and rejects the emulation with each of the mistakes a ragged kernel can make.

The launch: a 3x3 conv of 8 input channels into channels 0..7 of a 16-channel buffer (6 outputs and 2 pad lanes), at
half the network input's resolution, on a 64x96 canvas that holds a full frame and a 48x64 one.  Pooled, it has a ReLU
and a 2x2 max; unpooled, it is a head that also writes an fp32 map."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import ragged_check
from oracle import conv_check
from test_gpu_conv_tc_matrix import verdicts_for

H, W = 64, 96                       # network input
h, w = 32, 48                       # the launch's input
EXTS = [(64, 96), (48, 64)]
CIN, COUT, VALID, NT = 8, 16, 6, 8


def _bits(v):
    """bf16-valued float64 -> uint16 bit patterns."""
    return (v.to(torch.float32).numpy().view(np.uint32) >> 16).astype(np.uint16)


def _setup(pool):
    g = torch.Generator().manual_seed(5 + pool)
    sd = {"c.weight": (torch.rand((VALID, CIN, 3, 3), generator=g) - 0.5),
          "c.bias": (torch.rand(VALID, generator=g) - 0.5) * 0.1}
    t = dict(convs=["c"], in_ch=[np.arange(CIN)], off=[0], maps=[-1 if pool else 0], act="relu" if pool else None,
             slopes=[None])
    f = dict(ksize=3, cin_blocks=1, n_tile=NT, n_tiles=1, chunk=0, relu=int(pool), pool=pool, store0=NT)
    src = []
    for img, (he, we) in enumerate(EXTS):
        x = torch.zeros((h, w, CIN), dtype=torch.float64)
        x[:he // 2, :we // 2] = conv_check.bf16_round(torch.rand((he // 2, we // 2, CIN), generator=g) - 0.25)
        src.append(_bits(x))
    return sd, t, f, src


def emulate(sd, pool, src, exts, before):
    """The kernel on every image: a float64 convolution of the canvas input (what the kernel's loads see), rounded once
    to bf16 and to fp32, stored inside ext >> shift, +0 outside; pad lanes +0; channels 8..15 as they were."""
    ho_c, wo_c = (h // 2, w // 2) if pool else (h, w)
    w_hi = conv_check.split_weights(sd["c.weight"])[0]
    outs, maps = [], []
    for img, (x, ext) in enumerate(zip(src, exts)):
        xin = conv_check.bf16_to_f64(x).permute(2, 0, 1)[None]
        r = F.conv2d(xin, w_hi, sd["c.bias"].double(), padding=1)
        v = conv_check.bf16_round(conv_check.f_act(r, pool, pool))[0].permute(1, 2, 0)
        s = ragged_check.ext_shift(h, H, pool)
        ho, wo = ext[0] >> s, ext[1] >> s
        out = before[img].copy()
        out[..., :NT] = 0
        out[:ho, :wo, :VALID] = _bits(v[:ho, :wo])
        outs.append(out)
        m = np.zeros((VALID, ho_c, wo_c), np.float32)
        if not pool:                        # only the heads, which never pool, write fp32 maps
            m[:, :ho, :wo] = r[0, :, :ho, :wo].to(torch.float32).numpy()
        maps.append(m)
    return outs, maps


def verdict(sd, t, f, pool, src, after, before, maps):
    written = np.zeros(COUT, bool)
    written[:NT] = True
    fails, ratio = [], 0.0
    for img in range(len(EXTS)):
        fl, r = ragged_check.check_image(verdicts_for("bf16", sd, t, f, device="cpu"), [src[img]], [after[img]],
                                         [before[img]], EXTS[img], h, H, pool, written, [VALID, VALID + 1],
                                         [] if pool else [maps[img]], "image %d" % img)
        fails += fl
        ratio = max(ratio, r)
    return fails, ratio


MUTATIONS = ["outside_word", "outside_map", "neighbour_pad", "shift_up", "shift_down", "pad_lane", "slice"]


@pytest.mark.parametrize("pool", [0, 1])
def test_ragged_verdict_accepts_the_emulation_and_rejects_mistakes(pool):
    sd, t, f, src = _setup(pool)
    ho_c, wo_c = (h // 2, w // 2) if pool else (h, w)
    rs = np.random.RandomState(1)
    before = [rs.randint(0, 1 << 16, (ho_c, wo_c, COUT)).astype(np.uint16) for _ in EXTS]
    after, maps = emulate(sd, pool, src, EXTS, before)
    fails, ratio = verdict(sd, t, f, pool, src, after, before, maps)
    assert not fails, fails
    print("pool=%d: emulation %.3f of e" % (pool, ratio))
    (_, _), (ho, wo) = ragged_check.extents(EXTS[1], h, H, pool)
    for m in MUTATIONS:
        s2, a2, m2 = [x.copy() for x in src], [x.copy() for x in after], [x.copy() for x in maps]
        if m == "outside_word":             # one word just below the small frame
            a2[1][ho, 0, 2] = 0x0001
        elif m == "outside_map":
            if pool:
                continue
            m2[1][3, 0, wo] = np.float32(-0.0)
        elif m == "neighbour_pad":          # beyond the small frame, the canvas holds the full frame's pixels
            (hi, wi), _ = ragged_check.extents(EXTS[1], h, H, 0)
            s2[1][hi:] = src[0][hi:]
            s2[1][:hi, wi:] = src[0][:hi, wi:]
            a2, m2 = emulate(sd, pool, s2, EXTS, before)
        elif m in ("shift_up", "shift_down"):   # the extents one pooling level off
            d = 1 if m == "shift_up" else -1
            a2, m2 = emulate(sd, pool, src, [(e[0] >> d, e[1] >> d) if d > 0 else (e[0] << 1, e[1] << 1)
                                             for e in EXTS], before)
        elif m == "pad_lane":
            a2[0][0, 0, VALID + 1] = 0x8000     # -0 in a pad lane
        elif m == "slice":
            a2[0][5, 5, NT + 3] ^= 1
        got, _ = verdict(sd, t, f, pool, s2, a2, before, m2)
        print("pool=%d mutation %-14s %s" % (pool, m, "rejected: " + got[0].splitlines()[0] if got else "NOT visible"))
        assert got, m
