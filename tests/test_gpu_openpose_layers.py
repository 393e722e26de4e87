"""GPU (-m gpu): every launch of OpenPose_Model(l2, l1)'s bf16 and bf16x3 plans against a float64 reference of its own
inputs, as tests/test_gpu_layers.py does for rtpose, at the default layout (4, 2) and at layouts that (4, 2) does not
exercise: a PAF stage that is first and last (l2 = 1), a one-stage L1 branch (l1 = 1), a heat map feeding several later
stages (l1 >= 3) and all twelve outputs (l2 + l1 = 12).

The library's test hooks re-run the plan launch by launch and hand out each launch's real input and output planes and
its geometry.  Every element a launch writes is checked against the interval a correctly accumulated fp32 sum could
round to (oracle/conv_check.py; through a PReLU, tests/prelu_check.py's non-monotone rule), from a float64
convolution of the device's own bf16 inputs and weights derived from the state dict.  The head maps are checked in
fp32, pad channels must be exactly 0, and channels outside a launch's slice bit-unchanged."""
import time

import numpy as np
import pytest
import torch

import openpose_port
import prelu_check
from conftest import pkg_module
from oracle import conv_check

pytestmark = pytest.mark.gpu

L2, L1 = 4, 2
BUFS = ["t1", "t2", "t3", "t4", "t5a", "t5b", "t6", "t7", "t8", "t9", "cat", "bra", "brb", "br512"]
BUF = {b: i for i, b in enumerate(BUFS)}
BUF_C = [64, 64, 128, 128, 256, 256, 256, 512, 512, 256, 192, 768, 768, 512]     # OpenPose_Model's channel counts
BUF_DIV = [1, 2, 2, 4, 4, 4, 8, 8, 8, 8, 8, 8, 8, 8]
NUM_MAPS_BUF = len(BUFS)
FIELDS = ["in_buf", "in_cstride", "in_ch_base", "in_ch_group_stride", "out_buf", "out_cstride", "off0", "off1",
          "store0", "store1", "H", "W", "ksize", "cin_blocks", "groups", "n_tile", "n_tiles", "relu", "pool", "split",
          "chunk", "pdl", "tps", "map0", "map1", "n", "in_u8"]
REF = "cuda"
SHAPES = [((1, 8, 8), (0,)), ((2, 64, 72), (0, 1)), ((1, 184, 248), (0,)), ((1, 368, 368), (0,)),
          ((2, 368, 496), (0, 1)), ((8, 368, 368), (0, 7)), ((32, 368, 368), (0, 31))]
# (l2, l1) -> the shapes it runs: (4, 2) every shape of the rtpose check; the other layouts two small plans, (6, 6) also
# the one-frame plan at full resolution
LAYOUTS = {(4, 2): SHAPES, (1, 1): SHAPES[:2], (1, 11): SHAPES[:2], (11, 1): SHAPES[:2], (2, 3): SHAPES[:2],
           (6, 6): SHAPES[:2] + [SHAPES[3]]}
CASES = [(lay, s) for lay, shapes in LAYOUTS.items() for s in shapes]


def launch_table(l2=L2, l1=L1):
    """OpenPose_Model(l2, l1), per launch, in the reference's layer order: the conv's state-dict prefix, its activation ('relu', 'prelu' with the
    slope key, or none), the buffers, the physical input channels in the reference's channel order, the output channel
    offset and the fp32 map a head writes (DESIGN.md 2.11)."""
    spec = openpose_port.state_dict_spec(l2, l1)
    trunk = [k[:-len(".weight")] for k, s in spec.items() if k.startswith("feature_extractor.") and len(s) == 4]
    slope_of = {t: "feature_extractor.%d.weight" % (int(t.split(".")[1]) + 1) for t in trunk
                if "feature_extractor.%d.weight" % (int(t.split(".")[1]) + 1) in spec}
    T = [dict(conv=trunk[0], act="relu", slope=None, in_buf=-1, in_ch=np.arange(3), out_buf=BUF["t1"], off=0, pool=0,
              map=-1)]
    chain = [("t1", "t2", 1), ("t2", "t3", 0), ("t3", "t4", 1), ("t4", "t5a", 0), ("t5a", "t5b", 0), ("t5b", "t5a", 0),
             ("t5a", "t6", 1), ("t6", "t7", 0), ("t7", "t8", 0), ("t8", "t9", 0), ("t9", "cat", 0)]
    for i, (src, dst, pool) in enumerate(chain):
        c = trunk[i + 1]
        T.append(dict(conv=c, act="prelu" if c in slope_of else "relu", slope=slope_of.get(c), in_buf=BUF[src],
                      in_ch=np.arange(spec[c + ".weight"][1]), out_buf=BUF[dst], off=64 if dst == "cat" else 0,
                      pool=pool, map=-1))
    for t in range(l2 + l1):
        branch, i = ("l2", t) if t < l2 else ("l1", t - l2)
        _, inner, innerout, _ = openpose_port.stage_channels(branch, i)
        base = 384 if i == 0 else 0
        slots = np.concatenate([base + 128 * s + np.arange(inner) for s in range(3)])
        for li, (key, _, _, _, prelu) in enumerate(openpose_port.stage_convs(branch, i)):
            b, j = divmod(li, 3)
            cur, prev = ("bra", "brb") if b % 2 == 0 else ("brb", "bra")
            if li == 0:
                src, dst, off = "cat", cur, base
                in_ch = (np.arange(64, 192) if t == 0 else
                         np.r_[64:192, 0:38] if (branch == "l2" or i == 0) else np.r_[64:192, 40:59, 0:38])
            elif li < 15:
                src, dst = (prev, cur) if j == 0 else (cur, cur)
                in_ch = slots if j == 0 else base + 128 * (j - 1) + np.arange(inner)
                off = base + 128 * j
            elif li == 15:
                src, dst, off, in_ch = "bra", "br512", 0, slots
            else:
                src, dst, off, in_ch = "br512", "cat", 0 if branch == "l2" else 40, np.arange(innerout)
            T.append(dict(conv=key, act="prelu" if prelu else None,
                          slope=key[:-len(".Mconv")] + ".MPrelu.weight" if prelu else None, in_buf=BUF[src],
                          in_ch=in_ch, out_buf=BUF[dst], off=off, pool=0, map=t if li == 16 else -1))
    assert len(T) == 1 + 11 + 17 * (l2 + l1)
    return T


class Hooks:
    def __init__(self, net, l2=L2):
        self.l2 = l2
        self.nat = pkg_module("_native")
        self.lib = self.nat.lib()
        self.net = net

    def describe(self, i):
        f = np.zeros(len(FIELDS), np.int32)
        got = self.lib.b200pose_net_debug_launch(self.net._h, i, f.ctypes.data, len(f))
        assert got == len(FIELDS), self.lib.b200pose_last_error()
        return dict(zip(FIELDS, f.tolist()))

    def run(self, launches):
        self.nat.check(self.lib.b200pose_net_debug_run(self.net._h, launches, torch.cuda.current_stream().cuda_stream),
                       "b200pose_net_debug_run")

    def _read(self, buf, lo, img, shape, dtype):
        a = np.empty(shape, dtype)
        self.nat.check(self.lib.b200pose_net_debug_read(self.net._h, buf, lo, img, 1, a.ctypes.data, a.nbytes),
                       "b200pose_net_debug_read")
        return a

    def act(self, buf, lo, img, H, W):
        d = BUF_DIV[buf]
        return self._read(buf, lo, img, (H // d, W // d, BUF_C[buf]), np.uint16)

    def stage_map(self, m, img, H, W):
        return self._read(NUM_MAPS_BUF + m, 0, img, (38 if m < self.l2 else 19, H // 8, W // 8), np.float32)


def _nchw(u16, ch=None):
    t = conv_check.bf16_to_f64(u16, REF).permute(2, 0, 1)[None]
    return t if ch is None else t[:, torch.as_tensor(ch, device=REF)]


def check_plan(hooks, sd, x_in, n, H, W, imgs, mode, label, l2=L2, l1=L1):
    split = mode == "bf16x3"
    planes = (0, 1) if split else (0,)
    table = launch_table(l2, l1)
    fails, worst = [], {}
    before = None
    for i, t in enumerate(table):
        f = hooks.describe(i)
        ks = sd[t["conv"] + ".weight"].shape[2]
        div_in = 1 if t["in_buf"] < 0 else BUF_DIV[t["in_buf"]]
        want = dict(in_buf=t["in_buf"], out_buf=t["out_buf"], ksize=ks, relu=int(t["act"] == "relu"), pool=t["pool"],
                    groups=1, H=H // div_in, W=W // div_in, split=int(split), n=n, off0=t["off"], map0=t["map"])
        assert {k: f[k] for k in want} == want, "launch %d geometry %s, layer table %s" % (i, f, want)
        if i > 0:
            assert f["in_cstride"] == BUF_C[f["in_buf"]] and f["out_cstride"] == BUF_C[f["out_buf"]], (i, f)
            lib_ch = f["in_ch_base"] + np.arange(f["cin_blocks"] * 64)
            assert set(t["in_ch"]) <= set(lib_ch.tolist()), (i, f)
        hooks.run(i + 1)
        w32 = sd[t["conv"] + ".weight"]
        b = sd[t["conv"] + ".bias"].double().to(REF)
        valid, off = w32.shape[0], t["off"]
        kind = "conv1_1" if i == 0 else ("%s %dx%d N=%d" % (t["act"] or "head", ks, ks, f["n_tile"]))
        for img in imgs:
            after = [hooks.act(f["out_buf"], p, img, H, W) for p in planes]
            xin_lo = None
            if i == 0:
                xin = torch.from_numpy(x_in[img:img + 1].astype(np.float64)).to(REF)
                if not split:
                    xin = conv_check.bf16_round(xin)
            else:
                src = [hooks.act(f["in_buf"], p, img, H, W) for p in planes]
                xin = _nchw(src[0], t["in_ch"])
                xin_lo = _nchw(src[1], t["in_ch"]) if split else None
            if i == 0 and split:        # conv1_1 in bf16x3: fp32 CUDA-core FMA chain on the fp32 input and weights
                r, S = conv_check.reference(xin, w32.double().to(REF), b, ks)
                coef = conv_check.bound_coef(ks, 3, fma=True)
            else:
                w_hi, w_lo = conv_check.split_weights(w32)
                r, S = conv_check.reference(xin, w_hi.to(REF), b, ks, xin_lo, w_lo.to(REF) if split else None)
                coef = conv_check.bound_coef(ks, 3 if i == 0 else f["cin_blocks"] * 64, split=split and i > 0,
                                             chunk=bool(f["chunk"]))
            e = conv_check.U * coef * S
            where = "%s %s launch %d (%s, %s) image %d" % (label, mode, i, t["conv"], kind, img)
            got = _nchw(after[0][..., off:off + valid])
            got_lo = _nchw(after[1][..., off:off + valid]) if split else None
            if t["act"] == "prelu":
                slope = sd[t["slope"]].double()
                v = (prelu_check.check_split(got, got_lo, r, e, slope) if split else
                     prelu_check.check_bf16(got, r, e, slope))
            elif split:
                v = conv_check.check_split(got, got_lo, r, e, t["act"] == "relu", t["pool"])
            else:
                v = conv_check.check_bf16(got, r, e, t["act"] == "relu", t["pool"])
            if not bool(v.ok.all()):
                fails.append(conv_check.describe(v, got + got_lo if split else got, where, t["pool"]))
            worst[kind] = max(worst.get(kind, 0.0), v.ratio)
            if t["map"] >= 0:
                m = torch.from_numpy(hooks.stage_map(t["map"], img, H, W).astype(np.float64)).to(REF)[None]
                vm = conv_check.check_f32(m, r, e)
                if not bool(vm.ok.all()):
                    fails.append(conv_check.describe(vm, m, where + " fp32 map %d" % t["map"]))
                worst["head fp32 map"] = max(worst.get("head fp32 map", 0.0), vm.ratio)
            # channels the launch writes: per n-tile the first min(store, n_tile); beyond `valid` (head pads): 0
            store = min(f["store0"], f["n_tile"])
            written = np.zeros(BUF_C[f["out_buf"]], bool)
            for nt in range(f["n_tiles"]):
                written[off + nt * f["n_tile"]: off + nt * f["n_tile"] + store] = True
            pad = [int(c) for c in np.nonzero(written)[0] if c >= off + valid]
            for p in planes:
                if pad and np.any(after[p][..., pad]):
                    fails.append("%s: pad channels %s (plane %d) are not +0" % (where, pad, p))
            if before is not None:
                for p in planes:
                    if not np.array_equal(after[p][..., ~written], before[img][p][..., ~written]):
                        fails.append("%s: channels outside the launch's slice changed (plane %d)" % (where, p))
        if i + 1 < len(table):      # the next launch's output buffer as that launch finds it
            nb = hooks.describe(i + 1)["out_buf"]
            before = {img: [hooks.act(nb, p, img, H, W) for p in planes] for img in imgs}
    return fails, worst


@pytest.fixture(scope="module")
def layer_nets(built):
    """One net per layout, made when a test first asks for it."""
    nets = {}

    def get(l2, l1):
        if (l2, l1) not in nets:
            net = pkg_module("engine").NativeNet.openpose(0, l2, l1)
            sd = openpose_port.he_state_dict(l2, l1)
            net.load_state_dict_arrays([v.numpy() for v in sd.values()])
            nets.clear()            # one layout's buffers at a time
            nets[(l2, l1)] = net, sd
        return nets[(l2, l1)]
    return get


@pytest.mark.parametrize("mode", ["bf16", "bf16x3"])
@pytest.mark.parametrize("layout,shape,imgs", [(lay, s, i) for lay, (s, i) in CASES],
                         ids=[("%dx%dx%d" % s) if lay == (L2, L1) else ("%d-%d-%dx%dx%d" % (lay + s))
                              for lay, (s, _) in CASES])
def test_every_launch_matches_the_float64_reference(layer_nets, layout, shape, imgs, mode):
    l2, l1 = layout
    net, sd = layer_nets(l2, l1)
    nat = pkg_module("_native")
    t0 = time.time()
    n, H, W = shape
    x = torch.rand((n, 3, H, W), generator=torch.Generator().manual_seed(H * 1000 + W + n)) - 0.5
    xd = x.cuda().contiguous()
    net.forward_ptr(xd.data_ptr(), True, n, H, W, nat.MODES[mode], [0] * 12, True, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    label = "OpenPose_Model(%d, %d) %dx%dx%d" % (layout + shape)
    fails, worst = check_plan(Hooks(net, l2), sd, x.numpy(), n, H, W, imgs, mode, label, l2, l1)
    del xd
    print("\n%s %s: %d launches x %d image(s) checked in %.1f s; worst |v - r| / e per kind: %s" % (
        label, mode, len(launch_table(l2, l1)), len(imgs), time.time() - t0,
        "; ".join("%s %.3f" % kv for kv in sorted(worst.items()))))
    assert not fails, "\n".join(fails[:12]) + ("\n... %d failures in all" % len(fails) if len(fails) > 12 else "")
