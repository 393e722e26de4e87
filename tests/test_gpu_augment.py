"""GPU (-m gpu): training batches on the device (DESIGN.md 2.20; NativeNet.augment, PoseEngine.training_batch and
augmented_validation_loss).  training_batch equals the unmodified reference loader's samples (tests/golden/aug_*.npz)
bit for bit - images, heat and PAFs, flipped (float64 keypoints), JPEG and grayscale samples included - in ragged
mixed-size batches and alone, from host frames and from CUDA frames; the JPEG stage against the device encoder and
decoder; augmented_validation_loss against the composed path; refusals; launch counts."""
import numpy as np
import pytest
import torch

import aug_check as ac
from conftest import pkg_module

pytestmark = pytest.mark.gpu
GOLDENS = ac.goldens()


def _eng():
    return pkg_module("engine")


def _nat():
    return pkg_module("_native")


@pytest.fixture(scope="module")
def net(built, he_sd):
    n = _eng().NativeNet(0)
    n.load_state_dict_arrays([v.numpy() for v in he_sd.values()])
    return n


@pytest.fixture(scope="module")
def pe(net):
    return _eng().PoseEngine.from_net(net, mode="bf16", batch_cap=8)


def _bgr(g):
    return np.ascontiguousarray(g["src"][:, :, ::-1])


def _check(g, x, heat, paf):
    assert np.array_equal(ac.bits(x.cpu().numpy()), ac.bits(g["image"]))
    assert np.array_equal(ac.bits(heat.cpu().numpy()), ac.bits(g["heat"]))
    assert np.array_equal(ac.bits(paf.cpu().numpy()), ac.bits(g["paf"]))


@pytest.mark.parametrize("edge", [96, 368])
def test_training_batch_equals_every_golden(pe, edge):
    names = [k for k in sorted(GOLDENS) if int(GOLDENS[k]["edge"]) == edge]
    gs = [GOLDENS[k] for k in names]
    params = [ac.params_of(g)[0] for g in gs]
    x, heat, paf = pe.training_batch([_bgr(g) for g in gs], [g["kp"] for g in gs], edge=edge, params=params)
    torch.cuda.synchronize()
    assert x.shape == (len(gs), 3, edge, edge) and heat.shape == (len(gs), 19, edge // 8, edge // 8)
    for i, g in enumerate(gs):
        _check(g, x[i], heat[i], paf[i])


def test_each_ragged_sample_equals_itself_alone_from_cuda_frames(pe):
    """Every edge-96 golden alone, drawing from its own seeded generator, from a CUDA frame."""
    for name, g in sorted(GOLDENS.items()):
        if int(g["edge"]) != 96:
            continue
        src = torch.from_numpy(_bgr(g)).cuda()
        x, heat, paf = pe.training_batch([src], [g["kp"]], torch.Generator().manual_seed(int(g["seed"])), 96)
        _check(g, x[0], heat[0], paf[0])


def test_uint8_output_is_the_image_totensor_receives(net):
    gs = [g for g in GOLDENS.values() if int(g["edge"]) == 96]
    params = [ac.params_of(g)[0] for g in gs]
    x, u8 = net.augment([_bgr(g) for g in gs], params, 96, uint8=True)
    for i, g in enumerate(gs):
        assert np.array_equal(u8[i].cpu().numpy()[:, :, ::-1], g["u8"])


def test_jpeg_stage_equals_the_device_encoder_and_decoder(net):
    gs = [g for g in GOLDENS.values() if int(g["edge"]) == 96][:6]
    base = [dict(ac.params_of(g)[0], gray=False) for g in gs]
    frames = [_bgr(g) for g in gs]
    _, plain = net.augment(frames, [dict(p, jpeg=False) for p in base], 96, uint8=True)
    _, jpeg = net.augment(frames, [dict(p, jpeg=i % 2 == 0) for i, p in enumerate(base)], 96, uint8=True)
    want = net.decode_jpegs(net.encode_jpegs(plain, quality=50))
    for i in range(len(gs)):
        expect = want[i] if i % 2 == 0 else plain[i].cpu().numpy()
        assert np.array_equal(jpeg[i].cpu().numpy(), expect)


def test_augmented_validation_loss_equals_the_composed_path(pe):
    gs = [g for g in GOLDENS.values() if int(g["edge"]) == 96]
    images, kps = [_bgr(g) for g in gs], [g["kp"] for g in gs]
    got = pe.augmented_validation_loss(images, kps, torch.Generator().manual_seed(5), 96)
    gen = torch.Generator().manual_seed(5)
    sums, ext, cells = 0.0, [], 0
    stream = torch.cuda.current_stream().cuda_stream
    for at in range(0, len(gs), pe.post.batch_cap):
        x, heat, paf = pe.training_batch(images[at:at + 8], kps[at:at + 8], gen, 96)
        pe.net.forward_ptr(x.data_ptr(), True, x.shape[0], 96, 96, pe.mode, [None] * 12, True, stream)
        s, e, c, names = pe.net.stage_loss_sums(heat, paf)
        sums, cells = sums + s.sum(0), cells + sum(c)
        ext.append(e)
    want = _eng()._loss_dict(names, sums, np.concatenate(ext), cells)
    assert list(got) == list(want) and all(got[k] == want[k] for k in want)
    assert np.isfinite(got["total_loss"]) and got["total_loss"] > 0


def test_refusals_name_their_argument_and_leave_no_pending_error(net):
    eng, nat = _eng(), _nat()
    g = GOLDENS["small_flip"]
    p = ac.params_of(g)[0]
    frame = _bgr(g)
    bad = [
        (dict(p, order=[0, 0, 1, 2]), "permutation"),
        (dict(p, factors=(1.0, 1.0, 1.0, 0.7)), "hue"),
        (dict(p, resized=(1000, 10)), "resized"),
        (dict(p, crop=(5, 0)), "crop"),
        (dict(p, mask=(0, 0, 97, 96)), "mask"),
        (dict(p, jpeg=2), "0 or 1"),
    ]
    for q, what in bad:
        with pytest.raises(nat.B200PoseError, match=what):
            net.augment([frame], [q], 96)
    with pytest.raises(nat.B200PoseError, match="edge 100"):
        net.augment([frame], [dict(p, edge=100)], 100)
    with pytest.raises(nat.B200PoseError, match="size of image 0"):
        tiny = np.zeros((1, 5, 3), np.uint8)
        net.augment([tiny], [dict(p, size=(1, 5))], 96)
    with pytest.raises(nat.B200PoseError, match="params record"):
        net.augment([frame], [dict(p, size=(7, 7))], 96)
    torch.cuda.synchronize()
    x = net.augment([frame], [p], 96)
    torch.cuda.synchronize()
    assert np.array_equal(ac.bits(x[0].cpu().numpy()), ac.bits(g["image"]))
    with pytest.raises(nat.B200PoseError, match="not finite"):
        eng.ground_truth([np.full((1, 17, 3), np.nan)], [(96, 96)], 0, float64=True)


def test_launch_count_does_not_depend_on_n(net):
    nat = _nat()
    gs = [g for g in GOLDENS.values() if int(g["edge"]) == 96]
    counts = {}
    for jpeg in (False, True):
        for n in (1, 3, len(gs)):
            ps = [dict(ac.params_of(g)[0], jpeg=jpeg) for g in gs[:n]]
            l0 = nat.launch_count()
            net.augment([_bgr(g) for g in gs[:n]], ps, 96)
            counts.setdefault(jpeg, set()).add(nat.launch_count() - l0)
    assert counts[False] == {4}
    assert len(counts[True]) == 1 and counts[True].pop() > 4
