"""ORACLE (test infrastructure only).  The reference's second network, OpenPose_Model(l2, l1, 38, 19)
(/root/reference/lib/network/openpose.py:13-199), restated on the CPU:

  * state_dict_spec : its state_dict keys and shapes (module registration order);
  * he_state_dict   : seeded variance-preserving weights whose PReLU slopes include negative values and values above 1
                      (synthetic.openpose_state_dict; the reference's own init, normal(std=0.01) everywhere, makes every
                      map almost constant);
  * forward         : OpenPose_Model.forward with torch CPU ops (F.conv2d / F.prelu / torch.cat, the reference's own
                      arithmetic), pinned to the unmodified module by tests/golden/openpose_{64,368}.npz;
  * forward_exact   : the same graph on oracle/conv_exact.c (fp32, a defined accumulation order) with the PReLU applied
                      after the bias as one float32 multiply - what the product's fp32 mode computes bit for bit.

Maps come back in saved_for_loss order: [paf_1 .. paf_l2, heat_1 .. heat_l1], NCHW."""
from collections import OrderedDict

import numpy as np
import torch
import torch.nn.functional as F

PAF, HEAT, FEAT = 38, 19, 128
# make_vgg19_block: (name, cin, cout) per conv, 'P' = MaxPool2d(2, 2); PReLU after the last three convs
TRUNK = [("1_1", 3, 64), ("1_2", 64, 64), "P", ("2_1", 64, 128), ("2_2", 128, 128), "P", ("3_1", 128, 256),
         ("3_2", 256, 256), ("3_3", 256, 256), ("3_4", 256, 256), "P", ("4_1", 256, 512), ("4_2", 512, 512),
         ("4_3", 512, 256), ("4_4", 256, 128)]
TRUNK_PRELU = ("4_2", "4_3", "4_4")
BLOCKS = ["Mconv%d_%d" % (b, j) for b in range(1, 6) for j in range(3)]


def stage_channels(branch, i):
    """(in, inner, innerout, out) of stage i (0-based) of branch 'l2' / 'l1' (OpenPose_Model.__init__)."""
    first = i == 0
    if branch == "l2":
        cin = FEAT if first else FEAT + PAF
    else:
        cin = FEAT + PAF if first else FEAT + PAF + HEAT
    return cin, 96 if first else 128, 256 if first else 512, PAF if branch == "l2" else HEAT


def stage_convs(branch, i):
    """[(key prefix, cin, cout, k, prelu)] of one StageBlock."""
    cin, inner, innerout, out = stage_channels(branch, i)
    convs = []
    for n, blk in enumerate(BLOCKS):
        j = n % 3
        c = inner if j else (cin if n == 0 else 3 * inner)
        convs.append(("%s_stages.%d.%s.Mconv" % (branch, i, blk), c, inner, 3, True))
    convs.append(("%s_stages.%d.Mconv6.Mconv" % (branch, i), 3 * inner, innerout, 1, True))
    convs.append(("%s_stages.%d.Mconv7" % (branch, i), innerout, out, 1, False))
    return convs


def _slope_key(conv_key):
    """ConvBlock 'prefix.Mconv' -> its PReLU's 'prefix.MPrelu.weight'."""
    return conv_key[:-len(".Mconv")] + ".MPrelu.weight"


def state_dict_spec(l2=4, l1=2):
    spec = OrderedDict()
    idx = 0
    for item in TRUNK:
        if item == "P":
            idx += 1
            continue
        name, cin, cout = item
        spec["feature_extractor.%d.weight" % idx] = (cout, cin, 3, 3)
        spec["feature_extractor.%d.bias" % idx] = (cout,)
        if name in TRUNK_PRELU:
            spec["feature_extractor.%d.weight" % (idx + 1)] = (cout,)
        idx += 2
    for branch, count in (("l2", l2), ("l1", l1)):
        for i in range(count):
            for key, cin, cout, k, prelu in stage_convs(branch, i):
                spec[key + ".weight"] = (cout, cin, k, k)
                spec[key + ".bias"] = (cout,)
                if prelu:
                    spec[_slope_key(key)] = (cout,)
    return spec


def he_state_dict(l2=4, l1=2, seed=2024):
    """The seeded weights of the package's synthetic.openpose_state_dict (PReLU slopes in [-0.5, 1.5), He's gain for
    PReLU): the goldens were made with them, and tests/test_openpose_host.py checks its keys and shapes against the
    reference module's state_dict."""
    from conftest import pkg_module
    return pkg_module("synthetic").openpose_state_dict(l2, l1, seed)


def _trunk_keys():
    """[(weight key, bias key, slope key or None)] of the trunk's convs, in order, with the pools as 'P'."""
    out, idx = [], 0
    for item in TRUNK:
        if item == "P":
            out.append("P")
            idx += 1
            continue
        slope = "feature_extractor.%d.weight" % (idx + 1) if item[0] in TRUNK_PRELU else None
        out.append(("feature_extractor.%d.weight" % idx, "feature_extractor.%d.bias" % idx, slope))
        idx += 2
    return out


def forward(sd, x, l2=4, l1=2):
    """OpenPose_Model.forward (openpose.py:168-186) with torch CPU ops; x float32 [N,3,H,W] -> saved maps."""
    for item in _trunk_keys():
        if item == "P":
            x = F.max_pool2d(x, 2, 2, 0)
            continue
        wk, bk, sk = item
        x = F.conv2d(x, sd[wk], sd[bk], padding=1)
        x = F.prelu(x, sd[sk]) if sk else F.relu(x)
    features = x

    def stage(branch, i, y):
        outs = []
        for n, (key, _, _, k, prelu) in enumerate(stage_convs(branch, i)):
            if n < 15 and n % 3 == 0 and n > 0:
                y = torch.cat(outs[-3:], 1)
            elif n == 15:
                y = torch.cat(outs[-3:], 1)
            y = F.conv2d(y, sd[key + ".weight"], sd[key + ".bias"], padding=k // 2)
            if prelu:
                y = F.prelu(y, sd[_slope_key(key)])
            outs.append(y)
        return y

    saved, x_in = [], features
    for i in range(l2):
        paf = stage("l2", i, x_in)
        x_in = torch.cat([features, paf], 1)
        saved.append(paf)
    for i in range(l1):
        heat = stage("l1", i, x_in)
        x_in = torch.cat([features, heat, paf], 1)
        saved.append(heat)
    return saved


def prelu_f32(v, slope):
    """v > 0 ? v : slope * v, one float32 multiply (torch's CPU prelu); v NHWC float32."""
    s = np.asarray(slope, np.float32)
    return np.where(v > 0, v, (v * s).astype(np.float32))


def forward_exact(sd, x_nchw, l2=4, l1=2):
    """The same graph on oracle/conv_exact.c: every conv accumulates tap by tap, input channel by channel in the
    reference's concat order, adds the bias with one rounding, then ReLU or the PReLU above.  -> saved maps (NCHW)."""
    from oracle import net_exact
    g = lambda k: sd[k].numpy() if hasattr(sd[k], "numpy") else np.asarray(sd[k])
    x = np.ascontiguousarray(np.asarray(x_nchw, dtype=np.float32).transpose(0, 2, 3, 1))
    for item in _trunk_keys():
        if item == "P":
            x = net_exact.maxpool(x)
            continue
        wk, bk, sk = item
        x = net_exact.conv(x, g(wk), g(bk), sk is None)
        if sk:
            x = prelu_f32(x, g(sk))
    features = x
    n, h, w, _ = features.shape

    def conv(key, prelu, src, in_off, cin, out, out_off):
        y = net_exact.conv(src, g(key + ".weight"), g(key + ".bias"), False, in_off=in_off, cin=cin)
        if prelu:
            y = prelu_f32(y, g(_slope_key(key)))
        if out is not None:
            out[:, :, :, out_off:out_off + y.shape[3]] = y
        return y

    def stage(branch, i, x_in):
        _, inner, _, _ = stage_channels(branch, i)
        convs = stage_convs(branch, i)
        blk = [np.zeros((n, h, w, 3 * inner), np.float32) for _ in range(2)]
        for li in range(15):
            b, j = li // 3, li % 3
            key, cin, _, _, prelu = convs[li]
            dst = blk[b % 2]
            if li == 0:
                conv(key, prelu, x_in, 0, cin, dst, 0)
            elif j == 0:
                conv(key, prelu, blk[(b + 1) % 2], 0, cin, dst, 0)
            else:
                conv(key, prelu, dst, (j - 1) * inner, cin, dst, j * inner)
        y = conv(convs[15][0], True, blk[0], 0, 3 * inner, None, 0)
        return conv(convs[16][0], False, np.ascontiguousarray(y), 0, y.shape[3], None, 0)

    saved, x_in = [], features
    paf = None
    for i in range(l2):
        paf = stage("l2", i, x_in)
        x_in = np.ascontiguousarray(np.concatenate([features, paf], 3))
        saved.append(paf)
    for i in range(l1):
        heat = stage("l1", i, x_in)
        x_in = np.ascontiguousarray(np.concatenate([features, heat, paf], 3))
        saved.append(heat)
    return [np.ascontiguousarray(m.transpose(0, 3, 1, 2)) for m in saved]
