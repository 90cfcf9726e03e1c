"""BEV's streaming entry points on the GPU: forward_image_batches and forward_batches on the two-slot pipeline against
forward_images and forward_batch on a second instance, array for array, for plain, -t and --show_largest instances.
People are planted through center3d_override (synthetic weights)."""
import numpy as np
import pytest
import torch

from romp_b200 import synth
from romp_b200.bev import BEV, bev_settings
from romp_b200.main import img_preprocess

pytestmark = pytest.mark.gpu

MAX_BATCH = 4
SIZES = [(480, 640), (1080, 1920), (1280, 720), (512, 512), (300, 580), (720, 960)]


@pytest.fixture(scope="module")
def params():
    return synth.bev_damp_cam_offsets(synth.bev_state_dict(0)), synth.smpl_pack(0, num_betas=11), synth.smpl_pack(1)


def make(params, *flags):
    return BEV(bev_settings(["--max_batch", str(MAX_BATCH), *flags]), state_dict=params[0], smpla_pack=params[1],
               smil_pack=params[2])


def planted(n, seed, empty=(2,)):
    """3-D centre maps [n,64,128,128] of people who survive the post filters; frames in ``empty`` hold nobody."""
    vol, _ = synth.plant_centers_3d(n, seed=seed)
    vol[list(e for e in empty if e < n)] = 0.0
    return torch.from_numpy(vol).cuda()


def walkers(T, seed, people=8):
    """A seeded video [T,64,128,128]: people walking through the 3-D centre map, entering late and leaving early."""
    rs = np.random.RandomState(seed)
    vol = rs.uniform(0, 0.05, size=(T, 64, 128, 128)).astype(np.float32)
    for _ in range(people):
        t0, t1 = int(rs.randint(0, T // 3)), int(rs.randint(2 * T // 3, T + 1))
        p, v, val = rs.uniform([24, 16, 16], [44, 112, 112]), rs.uniform(-1.5, 1.5, 3) * [0, 1, 1], rs.uniform(0.3, 0.9)
        for t in range(t0, t1):
            z, y, x = np.clip(np.round(p + v * t), [0, 2, 2], [63, 125, 125]).astype(int)
            vol[t, z, y, x] = max(vol[t, z, y, x], val)
    return torch.from_numpy(vol).cuda()


def image(rs, k, where):
    h, w = SIZES[k % len(SIZES)]
    x = rs.randint(0, 256, (h, w, 3)).astype(np.uint8)
    return {"numpy": x, "host": torch.from_numpy(x), "device": torch.from_numpy(x).cuda()}[where]


def image_lists(seed, lengths, wide_in=None):
    """Lists of raw images of mixed sizes, as numpy arrays, host and device tensors; list ``wide_in`` also holds a
    1080x3840 crowd-mode image between its normal ones."""
    rs = np.random.RandomState(seed)
    lists = [[image(rs, k + n, ("numpy", "host", "device")[k % 3]) for k in range(n)] for n in lengths]
    if wide_in is not None:
        li = lists[wide_in]
        li.insert(len(li) // 2, rs.randint(0, 256, (1080, 3840, 3)).astype(np.uint8))
    return lists


def normal_count(li):
    return sum(1 for x in li if x.shape[1] / x.shape[0] < 2)


def host(x):
    return x.cpu().numpy() if isinstance(x, torch.Tensor) else x


def same(a, b, what):
    assert (a is None) == (b is None), what
    if a is None:
        return
    assert list(a) == list(b), (what, list(a), list(b))
    for k in a:
        x, y = host(a[k]), host(b[k])
        assert x.dtype == y.dtype and x.shape == y.shape and np.array_equal(x, y), (what, k)


def same_lists(got, ref):
    assert len(got) == len(ref)
    for i, (g, r) in enumerate(zip(got, ref)):
        assert len(g) == len(r), i
        for j, (a, b) in enumerate(zip(g, r)):
            same(a, b, (i, j))


LENGTHS = [0, 1, MAX_BATCH - 1, MAX_BATCH + 3]


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_image_batches_equal_forward_images(params, precision):
    m, m2 = make(params, "--precision", precision), make(params, "--precision", precision)
    lists = image_lists(1, LENGTHS, wide_in=3)
    vol = planted(MAX_BATCH + 3, 1)
    got = list(m.forward_image_batches(iter(lists), center3d_override=vol))
    ref = [m2.forward_images(li, center3d_override=vol[:normal_count(li)]) for li in lists]
    same_lists(got, ref)
    assert got[0] == [] and got[3][2] is None                                          # the frame planted empty
    assert all(r is not None for i, r in enumerate(got[3]) if i not in (2, 3))
    assert all(not r["pred_batch_ids"].any() for li in got for r in li if r is not None)
    dev = list(m.forward_image_batches(iter(lists), to_numpy=False, center3d_override=vol))
    assert isinstance(dev[3][0]["verts"], torch.Tensor) and dev[3][0]["verts"].is_cuda
    same_lists(dev, got)


def test_image_batches_without_smpl(params):
    m, m2 = make(params, "--precision", "fp32", "--calc_smpl"), make(params, "--precision", "fp32", "--calc_smpl")
    lists = image_lists(2, LENGTHS)
    vol = planted(MAX_BATCH + 3, 2)
    got = list(m.forward_image_batches(iter(lists), center3d_override=vol))
    same_lists(got, [m2.forward_images(li, center3d_override=vol[:len(li)]) for li in lists])
    assert "verts" not in got[3][0]


def test_frame_batches_equal_forward_batch(params):
    m, m2 = make(params, "--precision", "bf16"), make(params, "--precision", "bf16")
    batches = [synth.synthetic_frames(MAX_BATCH, seed=s) for s in range(3)]
    vol = planted(MAX_BATCH, 3, empty=())
    pads = np.stack([img_preprocess(np.zeros(SIZES[k] + (3,), np.uint8))[1] for k in range(MAX_BATCH)]).astype(np.float32)
    for offsets in (None, pads[0].tolist(), pads, torch.from_numpy(pads).cuda()):
        ref = [m2.forward_batch(b, offsets=offsets, center3d_override=vol, img_max_side=640.0) for b in batches]
        assert all(r is not None for r in ref)
        # the caller refills one pinned buffer as the generator pulls each batch, and scribbles on it after each yield
        buf = torch.empty((MAX_BATCH, 512, 512, 3), dtype=torch.uint8).pin_memory()

        def feed():
            for b in batches:
                buf.copy_(torch.from_numpy(b))
                yield buf
        got = []
        for r in m.forward_batches(feed(), offsets=offsets, center3d_override=vol, img_max_side=640.0):
            buf.fill_(7)
            got.append(r)
        same_lists([got], [ref])
        dev = list(m.forward_batches((torch.from_numpy(b).cuda() for b in batches), offsets=offsets, center3d_override=vol,
                                     img_max_side=640.0))
        same_lists([dev], [ref])


@pytest.mark.parametrize("mode", [["-t"], ["-t", "--show_largest"]])
def test_video_batches_equal_forward_images(params, mode):
    m, m2 = make(params, "--precision", "bf16", *mode), make(params, "--precision", "bf16", *mode)
    lengths = [3, 0, 9, 1, 7]
    for video in (5, 6):                                            # two videos, reset_temporal() between them
        lists = image_lists(video, lengths)
        sigs = [[(k // 2) % 2 for k in range(n)] for n in lengths]
        vol = walkers(max(lengths), video)
        got = list(m.forward_image_batches(iter(lists), center3d_override=vol, signal_IDs=iter(sigs)))
        ref = [m2.forward_images(li, center3d_override=vol[:len(li)], signal_IDs=s) for li, s in zip(lists, sigs)]
        same_lists(got, ref)
        assert m.frame_id == m2.frame_id
        out = [r for li in got for r in li if r is not None]
        assert len(out) > 10
        if "--show_largest" in mode:
            assert all(len(r["cam"]) <= 1 and len(r["params_pred"]) >= 1 for r in out)
        else:
            assert m.frame_id > 0
            assert min(int(r["track_ids"].min()) for r in out if len(r["track_ids"])) == 1
        m.reset_temporal()
        m2.reset_temporal()
