"""GPU (-m gpu): every launch of the bf16 and bf16x3 plans against a float64 reference of its own inputs.

The end-to-end bars (0.15 for bf16 over 52 layers of compounded rounding) cannot see a kernel that is subtly wrong in
one layer.  Here the library's test hooks re-run the plan launch by launch (b200pose_net_debug_run) and hand out each
launch's real input and output planes (b200pose_net_debug_read) and its geometry (b200pose_net_debug_launch).  Every
element every launch writes is checked with oracle/conv_check.py: the interval a correctly accumulated fp32 sum could
round to, from a float64 convolution of the device's own bf16 inputs and weights derived independently from the state
dict.  Channels outside a launch's slice must be bit-unchanged, the head slices' pad channels exactly 0.

The float64 references run on the GPU (cuDNN float64: float64 accumulation, 2^-25 below the bound, and cross-checked
against the CPU's float64 convolution on one launch below); the checks cost seconds, not CPU-minutes, per shape.
"""
import time

import numpy as np
import pytest
import torch

from conftest import pkg_module
from oracle import conv_check, glue_port, net_port

pytestmark = pytest.mark.gpu

BUFS = ["t1", "t2", "t3", "t4", "t5a", "t5b", "t6", "t7", "t8", "t9", "cat", "bra", "brb", "br512"]
BUF = {b: i for i, b in enumerate(BUFS)}
BUF_C = [64, 64, 128, 128, 256, 256, 256, 512, 512, 256, 192, 256, 256, 1024]
BUF_DIV = [1, 2, 2, 4, 4, 4, 8, 8, 8, 8, 8, 8, 8, 8]
NUM_MAPS_BUF = len(BUFS)            # debug_read ids 14 .. 25: the fp32 stage maps
FIELDS = ["in_buf", "in_cstride", "in_ch_base", "in_ch_group_stride", "out_buf", "out_cstride", "off0", "off1",
          "store0", "store1", "H", "W", "ksize", "cin_blocks", "groups", "n_tile", "n_tiles", "relu", "pool", "split",
          "chunk", "pdl", "tps", "map0", "map1", "n", "in_u8"]
# DESIGN.md section 1: physical channels of the concat buffer for torch.cat([paf 38, heat 19, features 128])
CAT_PHYS = np.r_[0:38, 40:59, 64:192]
REF = "cuda"

# (n, H, W), images checked
SHAPES = [((1, 8, 8), (0,)),            # 1x1 stage grid: every 7x7 tap but the centre in TMA zero-fill, pools down to 1x1
          ((2, 64, 72), (0, 1)),        # the suite's usual shape: 32-wide n-tiles, PDL
          ((1, 184, 248), (0,)),        # multi-scale 0.5x-like: odd 23 x 31 stage grid
          ((1, 368, 368), (0,)),        # small plan at full resolution: PDL, 64-wide stage n-tiles, pool at 92
          ((2, 368, 496), (0, 1)),      # raw 4:3 frame after crop_with_factor
          ((8, 368, 368), (0, 7)),      # large plan: N = 128, several tiles per CTA
          ((32, 368, 368), (0, 31))]    # the bench shape


def launch_table():
    """What each of the 52 launches computes, in the reference's layer order: per group the state-dict prefix of the
    conv and the physical input channels it reads; buffers, output channel offsets, ReLU, pool, fp32 maps."""
    spec = net_port.state_dict_spec()
    trunk = [k[:-len(".weight")] for k in spec if k.startswith("model0.") and k.endswith(".weight")]
    T = [dict(convs=[trunk[0]], in_buf=-1, in_ch=[np.arange(3)], out_buf=BUF["t1"], off=[0], relu=1, pool=0,
              maps=[-1])]
    chain = [("t1", "t2", 1), ("t2", "t3", 0), ("t3", "t4", 1), ("t4", "t5a", 0), ("t5a", "t5b", 0), ("t5b", "t5a", 0),
             ("t5a", "t6", 1), ("t6", "t7", 0), ("t7", "t8", 0), ("t8", "t9", 0), ("t9", "cat", 0)]
    for i, (src, dst, pool) in enumerate(chain):
        cin = spec[trunk[i + 1] + ".weight"][1]
        T.append(dict(convs=[trunk[i + 1]], in_buf=BUF[src], in_ch=[np.arange(cin)], out_buf=BUF[dst],
                      off=[64 if dst == "cat" else 0], relu=1, pool=pool, maps=[-1]))
    for s in range(1, 7):
        outs = ["bra", "brb", "bra", "br512", "cat"] if s == 1 else ["bra", "brb", "bra", "brb", "bra", "brb", "cat"]
        for li, dst in enumerate(outs):
            last = li == len(outs) - 1
            convs = ["model%d_%d.%d" % (s, br, 2 * li) for br in (1, 2)]
            cin = spec[convs[0] + ".weight"][1]
            if li == 0:
                src, in_ch = "cat", [np.arange(64, 192) if s == 1 else CAT_PHYS] * 2
            else:
                src = outs[li - 1]
                width = 512 if src == "br512" else 128
                in_ch = [g * width + np.arange(cin) for g in (0, 1)]
            off = [0, 40] if dst == "cat" else ([0, 512] if dst == "br512" else [0, 128])
            T.append(dict(convs=convs, in_buf=BUF[src], in_ch=in_ch, out_buf=BUF[dst], off=off, relu=0 if last else 1,
                          pool=0, maps=[2 * (s - 1), 2 * (s - 1) + 1] if last else [-1, -1]))
    assert len(T) == 52
    return T


class Hooks:
    def __init__(self, net):
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
        """uint16 [h, w, C] bf16 bits of one image of activation buffer `buf` (H, W: network input size)."""
        d = BUF_DIV[buf]
        return self._read(buf, lo, img, (H // d, W // d, BUF_C[buf]), np.uint16)

    def stage_map(self, m, img, H, W):
        return self._read(NUM_MAPS_BUF + m, 0, img, (38 if m % 2 == 0 else 19, H // 8, W // 8), np.float32)


def _nchw(u16, ch=None):
    t = conv_check.bf16_to_f64(u16, REF).permute(2, 0, 1)[None]
    return t if ch is None else t[:, torch.as_tensor(ch, device=REF)]


def _variant(f):
    if f["ksize"] == 3 and f["in_buf"] < 0:
        return "conv1_1 " + ("fp32 FMA (bf16x3)" if f["split"] else "mma.sync (bf16)")
    return "wgmma N=%d %s" % (f["n_tile"], "chunked" if f["chunk"] else "unchunked")


def check_plan(hooks, sd, x_in, n, H, W, imgs, mode, launches=52, label=""):
    """Checks the first `launches` launches of the plan the last forward built.  x_in: the network input as the kernels
    see it after normalisation, float32 numpy [n, 3, H, W].  Returns (failure messages, per-launch report rows)."""
    split = mode == "bf16x3"
    planes = (0, 1) if split else (0,)
    table = launch_table()
    num_sms = torch.cuda.get_device_properties(0).multi_processor_count
    fails, rows = [], []
    before = None
    for i in range(launches):
        f, t = hooks.describe(i), table[i]
        # ---- the geometry the library reports agrees with the reference's layer table
        ks = sd[t["convs"][0] + ".weight"].shape[2]
        div_in = 1 if t["in_buf"] < 0 else BUF_DIV[t["in_buf"]]
        want = dict(in_buf=t["in_buf"], out_buf=t["out_buf"], ksize=ks, relu=t["relu"], pool=t["pool"],
                    groups=len(t["convs"]), H=H // div_in, W=W // div_in, split=int(split), n=n,
                    off0=t["off"][0], map0=t["maps"][0])
        if len(t["convs"]) == 2:
            want.update(off1=t["off"][1], map1=t["maps"][1])
        assert {k: f[k] for k in want} == want, "launch %d geometry %s, layer table %s" % (i, f, want)
        if i > 0:
            assert f["in_cstride"] == BUF_C[f["in_buf"]] and f["out_cstride"] == BUF_C[f["out_buf"]], (i, f)
            for g in range(f["groups"]):
                lib_ch = f["in_ch_base"] + g * f["in_ch_group_stride"] + np.arange(f["cin_blocks"] * 64)
                assert set(t["in_ch"][g]) <= set(lib_ch.tolist()) and len(lib_ch) == 64 * -(-len(t["in_ch"][g]) // 64), \
                    (i, g, f)
        hooks.run(i + 1)
        h, w = f["H"], f["W"]
        ho, wo = (h // 2, w // 2) if f["pool"] else (h, w)
        tiles = n * -(-h // 16) * -(-w // 8) * f["groups"] * f["n_tiles"]
        row = dict(launch=i, conv=t["convs"][0], variant=_variant(f), pdl=f["pdl"], tiles=tiles,
                   tiles_per_cta=-(-tiles // num_sms), ratio_out=0.0, ratio_map=None)
        for img in imgs:
            after = [hooks.act(f["out_buf"], p, img, H, W) for p in planes]
            if i == 0:
                xin = torch.from_numpy(x_in[img:img + 1].astype(np.float64)).to(REF)
                xin_lo = None
                if not split:
                    xin = conv_check.bf16_round(xin)
            else:
                src = [hooks.act(f["in_buf"], p, img, H, W) for p in planes]
            written = np.zeros(BUF_C[f["out_buf"]], bool)
            for g, conv in enumerate(t["convs"]):
                w32 = sd[conv + ".weight"]
                b = sd[conv + ".bias"].double().to(REF)
                valid = w32.shape[0]
                if i > 0:
                    xin = _nchw(src[0], t["in_ch"][g])
                    xin_lo = _nchw(src[1], t["in_ch"][g]) if split else None
                if i == 0 and split:        # fp32 CUDA-core FMA chain on the fp32 input and weights
                    r, S = conv_check.reference(xin, w32.double().to(REF), b, ks)
                    coef = conv_check.bound_coef(ks, 3, fma=True)
                else:
                    w_hi, w_lo = conv_check.split_weights(w32)
                    r, S = conv_check.reference(xin, w_hi.to(REF), b, ks, xin_lo, w_lo.to(REF) if split else None)
                    coef = conv_check.bound_coef(ks, 3 if i == 0 else f["cin_blocks"] * 64, split=split and i > 0,
                                                 chunk=bool(f["chunk"]))
                e = conv_check.U * coef * S
                off = t["off"][g]
                where = "%s %s launch %d (%s, %s) image %d group %d" % (label, mode, i, conv, row["variant"], img, g)
                got = _nchw(after[0][..., off:off + valid])
                if split:
                    got_lo = _nchw(after[1][..., off:off + valid])
                    v = conv_check.check_split(got, got_lo, r, e, f["relu"], f["pool"])
                else:
                    v = conv_check.check_bf16(got, r, e, f["relu"], f["pool"])
                if not bool(v.ok.all()):
                    fails.append(conv_check.describe(v, got + got_lo if split else got, where, f["pool"]))
                row["ratio_out"] = max(row["ratio_out"], v.ratio)
                if t["maps"][g] >= 0:
                    m = torch.from_numpy(hooks.stage_map(t["maps"][g], img, H, W).astype(np.float64)).to(REF)[None]
                    vm = conv_check.check_f32(m, r, e)
                    if not bool(vm.ok.all()):
                        fails.append(conv_check.describe(vm, m, where + " fp32 map %d" % t["maps"][g]))
                    row["ratio_map"] = max(row["ratio_map"] or 0.0, vm.ratio)
                # channels this group writes: per n-tile the first min(store_ch, n_tile); beyond `valid` (head pads): 0
                store = min(f["store%d" % g], f["n_tile"])
                mine = np.zeros_like(written)
                for nt in range(f["n_tiles"]):
                    mine[off + nt * f["n_tile"]: off + nt * f["n_tile"] + store] = True
                written |= mine
                pad = [int(c) for c in np.nonzero(mine)[0] if c >= off + valid]
                for p in planes:
                    if pad and np.any(after[p][..., pad] & 0x7FFF):
                        fails.append("%s: pad channels %s (plane %d) are not 0" % (where, pad, p))
            if before is not None and not written.all():
                for p in planes:
                    if not np.array_equal(after[p][..., ~written], before[img][p][..., ~written]):
                        fails.append("%s %s launch %d image %d: channels outside the launch's slice changed (plane %d)"
                                     % (label, mode, i, img, p))
        rows.append(row)
        if i + 1 < launches:    # the next launch's output buffer as that launch finds it
            nb = hooks.describe(i + 1)["out_buf"]
            before = {img: [hooks.act(nb, p, img, H, W) for p in planes] for img in imgs}
    return fails, rows


def _report(rows, label):
    print("\n%s: per-launch max |v - r| / e (bf16 outputs: distance to the rounding cell of the returned value; "
          "fp32 maps: exact)" % label)
    for r in rows:
        print("  launch %2d %-16s %-26s pdl=%d tiles=%5d tiles/CTA=%3d  out %.3f%s" % (
            r["launch"], r["conv"], r["variant"], r["pdl"], r["tiles"], r["tiles_per_cta"], r["ratio_out"],
            "" if r["ratio_map"] is None else "  map %.3f" % r["ratio_map"]))
    worst = {}
    for r in rows:
        key = r["variant"]
        worst[key] = max(worst.get(key, 0.0), r["ratio_out"], r["ratio_map"] or 0.0)
    print("  worst per variant: " + "; ".join("%s %.3f" % kv for kv in sorted(worst.items())))
    print("  PDL launches: %s" % [r["launch"] for r in rows if r["pdl"]])


@pytest.fixture(scope="module")
def layer_net(built, he_sd):
    eng = pkg_module("engine")
    net = eng.NativeNet(0)
    net.load_state_dict_arrays([v.numpy() for v in he_sd.values()])
    return net


def _forward(net, x, mode):
    nat = pkg_module("_native")
    n, _, H, W = x.shape
    xd = x.cuda().contiguous()
    net.forward_ptr(xd.data_ptr(), True, n, H, W, nat.MODES[mode], [0] * 12, True, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return xd          # the hooks re-run the plan on this buffer: keep it alive


@pytest.mark.parametrize("mode", ["bf16", "bf16x3"])
@pytest.mark.parametrize("shape,imgs", SHAPES, ids=["%dx%dx%d" % s for s, _ in SHAPES])
def test_every_launch_matches_the_float64_reference(layer_net, he_sd, shape, imgs, mode):
    t0 = time.time()
    n, H, W = shape
    x = torch.rand((n, 3, H, W), generator=torch.Generator().manual_seed(H * 1000 + W + n)) - 0.5
    xd = _forward(layer_net, x, mode)
    label = "%dx%dx%d" % shape
    fails, rows = check_plan(Hooks(layer_net), he_sd, x.numpy(), n, H, W, imgs, mode, label=label)
    del xd
    _report(rows, "%s %s" % (label, mode))
    print("%s %s: 52 launches x %d image(s) checked in %.1f s" % (label, mode, len(imgs), time.time() - t0))
    assert not fails, "\n".join(fails[:12]) + ("\n... %d failures in all" % len(fails) if len(fails) > 12 else "")


@pytest.mark.parametrize("mode", ["bf16", "bf16x3"])
@pytest.mark.parametrize("pre", ["rtpose", "vgg"])
def test_conv1_1_on_uint8_frames(layer_net, he_sd, pre, mode):
    """conv1_1 with the normalisation fused into its load.  rtpose values are exact in bf16; vgg's are not, so the
    bf16 reference operand is bf16(vgg_preprocess(u8)) (bf16x3: the fp32 value itself)."""
    nat = pkg_module("_native")
    img = np.random.RandomState(5).randint(0, 256, (2, 64, 72, 3)).astype(np.uint8)
    prep = {"rtpose": glue_port.rtpose_preprocess, "vgg": glue_port.vgg_preprocess}[pre]
    x = np.stack([prep(i) for i in img])
    if pre == "rtpose":
        assert np.array_equal(conv_check.bf16_round(torch.from_numpy(x.astype(np.float64))).numpy(), x)
    layer_net.set_preprocess(pre)
    try:
        xd = torch.from_numpy(img).cuda()
        layer_net.forward_u8_ptr(xd.data_ptr(), True, 2, 64, 72, nat.MODES[mode], [0] * 12, True,
                                 torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        hooks = Hooks(layer_net)
        assert hooks.describe(0)["in_u8"] == nat.PREPROCESS[pre]
        fails, rows = check_plan(hooks, he_sd, x, 2, 64, 72, (0, 1), mode, launches=1, label="u8 " + pre)
    finally:
        layer_net.set_preprocess("rtpose")
    print("conv1_1 %s %s: max |v - r| / e %.3f" % (pre, mode, rows[0]["ratio_out"]))
    assert not fails, "\n".join(fails[:12])


def test_gpu_float64_reference_equals_the_cpu_one(he_sd):
    """The float64 references above run on the GPU; on one 7x7 Mconv1 they agree with the CPU's to far below the
    bound (float64 accumulation: relative error ~1e-16)."""
    w_hi, w_lo = conv_check.split_weights(he_sd["model2_1.0.weight"])
    b = he_sd["model2_1.0.bias"].double()
    x = conv_check.bf16_round(torch.rand((1, 185, 23, 31), generator=torch.Generator().manual_seed(1), dtype=torch.float64))
    r_c, s_c = conv_check.reference(x, w_hi, b, 7)
    r_g, s_g = conv_check.reference(x.cuda(), w_hi.cuda(), b.cuda(), 7)
    assert float(((r_g.cpu() - r_c).abs() / s_c).max()) < 1e-12
    assert float(((s_g.cpu() - s_c).abs() / s_c).max()) < 1e-12
