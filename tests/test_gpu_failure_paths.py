"""GPU (-m gpu): recovery after a failed call.  A post object whose creation runs out of device memory raises, and
leaves no CUDA error behind that would fail the next call on the same host thread; the objects created before and after
it work as if the failed call had not happened."""
import pytest
import torch

from conftest import POST_CASES, assert_humans_equal, golden, humans_rows_to_dicts, pkg_module
from oracle import synth

pytestmark = pytest.mark.gpu

# post_alloc's first buffer (per-image part counts, 75.5 MB) fits; its second (peak x coordinates, 1 Mi x 18 x 2048 x 4
# bytes = 154.6 GB) is larger than the card, so the create fails at once and reserves nothing large.
TOO_BIG = dict(batch_cap=1 << 20, peak_cap=2048, human_cap=16)
TOO_BIG_BYTES = (1 << 20) * 18 * 2048 * 4


def _failed_create(eng, nat):
    with pytest.raises(nat.B200PoseError, match="post_alloc"):
        eng.NativePost(0, **TOO_BIG)


def _post_p3_matches_golden(eng):
    """A normal post object: create, run on the p3 maps, compare with the reference's humans, destroy."""
    heat, paf = POST_CASES["p3"](synth)
    h, w = heat.shape[:2]
    post = eng.NativePost(0, batch_cap=1, peak_cap=1024, human_cap=1024)
    post.run(heat.ctypes.data, paf.ctypes.data, False, 1, 1, h, w, 0.1)
    post.sync()
    post.check_status(1)
    got = eng.humans_to_dicts(post.humans(0), w * 8, h * 8)
    assert_humans_equal(got, humans_rows_to_dicts(golden("post_p3")["humans"]), score_tol=1e-6)
    del post
    torch.cuda.synchronize()


@pytest.fixture
def post_oom_possible(built):
    if torch.cuda.get_device_properties(0).total_memory >= TOO_BIG_BYTES:
        pytest.skip("the device could hold the oversized request")


def test_failed_create_leaves_no_error_for_the_next_call(post_oom_possible, he_sd):
    eng, nat = pkg_module("engine"), pkg_module("_native")
    net = eng.NativeNet(0)
    net.load_state_dict_arrays([v.numpy() for v in he_sd.values()])
    x = (torch.rand((2, 3, 64, 64), generator=torch.Generator().manual_seed(3)) - 0.5).cuda()
    outs = [[torch.empty((2, 38 if i % 2 == 0 else 19, 8, 8), device="cuda") for i in range(12)] for _ in range(2)]
    stream = torch.cuda.current_stream().cuda_stream

    def forward(o):
        net.forward_ptr(x.data_ptr(), True, 2, 64, 64, nat.MODES["bf16"], [t.data_ptr() for t in o], True, stream)

    forward(outs[0])
    torch.cuda.synchronize()
    _failed_create(eng, nat)
    # same host thread and no torch CUDA call in between (torch's launch checks would consume a pending error)
    forward(outs[1])
    torch.cuda.synchronize()
    for i, (a, b) in enumerate(zip(*outs)):
        assert torch.equal(a, b), "map %d differs after the failed create" % i
    _post_p3_matches_golden(eng)


def test_repeated_failed_creates(post_oom_possible):
    eng, nat = pkg_module("engine"), pkg_module("_native")
    for _ in range(8):
        _failed_create(eng, nat)
    _post_p3_matches_golden(eng)
