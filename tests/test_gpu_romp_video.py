"""ROMP's batched video mode (ROMP.forward_video, csrc/romp_track.cu) against the per-frame temporal path it batches.

1. The track step through the C ABI, fed seeded cam sequences without a model, against TemporalState.assign frame by
   frame (slots, track ids, row counts exactly) and b200romp_one_euro_smooth driven with the host's slots and resets;
   the same sequence cut into batches of 1, 7 and 64 gives bit-identical results.
2. forward_video on a fresh instance against [forward(img) for img in images] on another, end to end.
3. forward_video_batches against forward_video; planted moving people and empty frames against the plain
   forward_images post-processed by TemporalState and the oracle recurrences (oracle/temporal_oracle.py).
4. The API rules: reset_temporal(), forward / forward_video mixing, signal_IDs length."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import preproc_oracle as P
from oracle import romp_oracle as O
from oracle import temporal_oracle as TO
from romp_b200 import ROMP, _lib, romp_settings, synth
from romp_b200.temporal import TemporalState

pytestmark = pytest.mark.gpu


def _p(t):
    return C.c_void_p(t.data_ptr())


# ------------------------------------------------------------------------------------------------
# 1. the track step against TemporalState + b200romp_one_euro_smooth
# ------------------------------------------------------------------------------------------------
def cam_of(px):
    """points cam[:,[2,1]] * 512 = px (integer pixels: exact in fp32) -> cam rows with scale 1."""
    px = np.asarray(px, np.float64).reshape(-1, 2)
    cam = np.ones((len(px), 3), np.float32)
    cam[:, 2], cam[:, 1] = px[:, 0] / 512.0, px[:, 1] / 512.0
    return cam


def stage_sequence():
    """[(cam [n,3] float32, signal_ID)] covering the cases the tracker distinguishes."""
    rs = np.random.RandomState(11)
    seq = []
    # random walks of 1..64 people, in a random detection order
    pos = rs.uniform(-600, 600, (64, 2))
    for _ in range(40):
        pos += rs.normal(0, 25, pos.shape)
        k = rs.randint(1, 65)
        idx = rs.permutation(64)[:k]
        cam = cam_of(np.round(pos[idx]))
        cam[:, 0] = rs.uniform(0.5, 1.5, k)
        seq.append((cam, 0))
    # an empty frame, then one person absent for 35 frames while another stays; the first one returns with a new id
    seq.append((np.zeros((0, 3), np.float32), 0))
    seq.append((cam_of([[5000, 5000], [-5000, -5000]]), 1))
    for t in range(35):
        seq.append((cam_of([[-5000, -5000 + t]]), 1))
        if t % 9 == 4:
            seq.append((np.zeros((0, 3), np.float32), 1))
    seq.append((cam_of([[5000, 5000], [-5000, -4966]]), 1))
    # two detections within 200 px of one track; a detection exactly 200 px away starts a new track
    seq.append((cam_of([[0, 3000]]), 2))
    seq.append((cam_of([[10, 3000], [20, 3000], [220, 3000]]), 2))
    # symmetric tracks at x -+ 3 (track 2 walks in on its side of the bisector), then a detection at x: the earlier track
    for g in [200, 98, 47, 21, 8, 2, 0]:
        seq.append((cam_of([[-3, -3000], [3 + g, -3000]]), 3))
    seq.append((cam_of([[0, -3000]]), 3))
    seq.append((cam_of([[0, -3000], [-3, -3000], [3, -3000]]), 3))
    # more than 64 concurrent tracks: 64 scattered new people per frame for 33 frames (up to 31 x 64 live tracks, slots
    # run out, rows stay unsmoothed, slots come back as tracks age out)
    for _ in range(33):
        cam = cam_of(np.round(rs.uniform(-10000, 10000, (64, 2))))
        seq.append((cam, 4))
    # 5-6 signals interleaved (eviction of the earliest registered, block reset, ids restarting), empty frames among them
    for t in range(24):
        sid = [5, 6, 7, 8, 9, 5, 10, 6][t % 8]
        n = (t * 5) % 7
        seq.append((cam_of(np.round(rs.uniform(-400, 400, (n, 2)))), sid))
    # --show_largest ties: two rows with the same scale
    cam = cam_of([[0, 0], [500, 0], [-500, 0]])
    cam[:, 0] = [0.7, 1.3, 1.3]
    seq.append((cam, 0))
    return seq


def add_params(seq, seed=5):
    rs = np.random.RandomState(seed)
    out = []
    for cam, sid in seq:
        n = len(cam)
        th = rs.normal(0, 0.4, (n, 72)).astype(np.float32)
        be = rs.normal(0, 1.0, (n, 10)).astype(np.float32)
        out.append((cam, th, be, sid))
    return out


def host_path(frames, largest):
    """TemporalState.assign + b200romp_one_euro_smooth per frame (forward's temporal path without the model)."""
    lib, st = _lib.load(), C.c_void_p(torch.cuda.current_stream().cuda_stream)
    ts = TemporalState(largest)
    h = lib.b200romp_tracks_create(0, ts.n_slots)
    assert h
    res = []
    for cam, th, be, sid in frames:
        n = len(cam)
        if n == 0:
            res.append(None)
            continue
        slots, ids, reset = ts.assign(cam, sid)
        for sl in reset:
            _lib.check(lib.b200romp_tracks_reset(h, int(sl), st))
        d = [torch.from_numpy(x.copy()).cuda() for x in (slots, th, be, cam)]
        _lib.check(lib.b200romp_one_euro_smooth(h, _p(d[0]), n, None, _p(d[1]), _p(d[2]), 10, 10, _p(d[3]), 3.0, 30.0,
                                                int(not largest), st))
        s_th, s_be, s_cam = (x.cpu().numpy() for x in d[1:])
        if largest:
            k = int(np.argmax(cam[:, 0]))
            s_th, s_be, s_cam = s_th[k:k + 1], s_be[k:k + 1], s_cam[k:k + 1]
        res.append(dict(slot=slots, ids=ids, thetas=s_th, betas=s_be, cam=s_cam))
    lib.b200romp_tracks_destroy(h)
    return res


def device_path(frames, largest, batch):
    """b200romp_romp_track_step over the frames in batches of ``batch``."""
    lib, st = _lib.load(), C.c_void_p(torch.cuda.current_stream().cuda_stream)
    h = lib.b200romp_romp_tracker_create(0, 4)
    assert h
    codes = {}
    res = []
    cap = batch * 64
    z = lambda *s, dt=torch.float32: torch.zeros(*s, dtype=dt, device="cuda")
    o = dict(count=z(1, dt=torch.int32), ids=z(cap, dt=torch.int64), thetas=z(cap, 72), betas=z(cap, 10), cam=z(cap, 3),
             slot=z(cap, dt=torch.int32), track=z(cap, dt=torch.int32))
    cam, th, be, ids = z(cap, 3), z(cap, 72), z(cap, 10), z(cap, dt=torch.int64)
    for c0 in range(0, len(frames), batch):
        ch = frames[c0:c0 + batch]
        B = len(ch)
        ns = [len(f[0]) for f in ch]
        N = sum(ns)
        cat = lambda i, w: torch.from_numpy(np.concatenate([f[i] for f in ch]).reshape(-1, w))
        cam[:N], th[:N], be[:N] = cat(0, 3), cat(1, 72), cat(2, 10)
        ids[:N] = torch.from_numpy(np.repeat(np.arange(B), ns).astype(np.int64))
        cnt = torch.tensor([N], dtype=torch.int32, device="cuda")
        sig = torch.tensor([codes.setdefault(f[3], len(codes)) for f in ch], dtype=torch.int32, device="cuda")
        th0 = th.clone()
        _lib.check(lib.b200romp_romp_track_step(h, B, cap, _p(cnt), _p(ids), _p(cam), _p(th), _p(be), _p(sig), int(largest), 3.0,
                                                30.0, _p(o["count"]), _p(o["ids"]), _p(o["thetas"]), _p(o["betas"]), _p(o["cam"]),
                                                _p(o["slot"]), _p(o["track"]), st), "romp_track_step")
        torch.cuda.synchronize()
        assert torch.equal(th, th0)                      # the inputs are left as they are
        m = int(o["count"].item())
        assert m == (sum(n > 0 for n in ns) if largest else sum(ns))
        h_ = {k: v.cpu().numpy() for k, v in o.items()}
        r0, j = 0, 0
        for b, n in enumerate(ns):
            if n == 0:
                res.append(None)
                continue
            rows = slice(j, j + 1) if largest else slice(r0, r0 + n)
            assert np.all(h_["ids"][rows] == b)
            res.append(dict(slot=h_["slot"][r0:r0 + n].copy(), ids=None if largest else h_["track"][r0:r0 + n].copy(),
                            thetas=h_["thetas"][rows].copy(), betas=h_["betas"][rows].copy(), cam=h_["cam"][rows].copy()))
            r0 += n
            j += 1
    lib.b200romp_romp_tracker_destroy(h)
    return res


@pytest.mark.parametrize("largest", [False, True])
def test_track_step_matches_temporal_state(largest):
    frames = add_params(stage_sequence())
    ref = host_path(frames, largest)
    if not largest:      # the sequence reaches the cases it is built for
        ids = [r["ids"] for r in ref if r is not None]
        assert any(np.any(r["slot"] == -1) and len(r["slot"]) == 64 for r in ref if r is not None)   # slots ran out
        assert any(len(set(i.tolist())) < len(i) for i in ids)                                      # two rows, one track
        assert max(int(i.max()) for i in ids) > 64 * 20                                             # many tracks
    runs = {b: device_path(frames, largest, b) for b in (1, 7, 64)}
    err = 0.0
    for t, r in enumerate(ref):
        for b, res in runs.items():
            g = res[t]
            assert (g is None) == (r is None), (b, t)
            if r is None:
                continue
            assert np.array_equal(g["slot"], r["slot"]), (b, t)
            if not largest:
                assert np.array_equal(g["ids"], r["ids"]), (b, t)
            assert len(g["cam"]) == len(r["cam"]), (b, t)
            for k in ("thetas", "betas", "cam"):
                err = max(err, float(np.abs(g[k] - r[k]).max()))
                assert np.array_equal(g[k], runs[1][t][k]), (b, t, k)      # bit-identical across batch sizes
    print(f"largest={largest}: max |track step - host path| = {err:.2e} over {len(ref)} frames")
    assert err < 3e-5


def test_track_step_exact_cases():
    """The tie, the 200-px boundary and the returning person, read off the device ids directly."""
    frames = add_params(stage_sequence())
    res = device_path(frames, False, 64)
    by_sig = {}
    for f, r in zip(frames, res):
        if r is not None:
            by_sig.setdefault(f[3], []).append(r["ids"])
    s2 = by_sig[2]
    assert s2[0].tolist() == [1] and s2[1].tolist() == [1, 1, 2]        # both within 200 px of track 1; 200 px: new track
    s3 = by_sig[3]
    assert s3[-3].tolist() == [1, 2]                                  # the walk kept the two tracks apart
    assert s3[-2].tolist() == [1] and s3[-1].tolist() == [1, 1, 2]    # tie -> the earlier track
    s1 = by_sig[1]
    assert s1[0].tolist() == [1, 2] and s1[-1].tolist() == [3, 2]     # absent > 30 frames: a new id
    assert max(len(i) for i in by_sig[4]) == 64


# ------------------------------------------------------------------------------------------------
# 2./3./4. ROMP.forward_video
# ------------------------------------------------------------------------------------------------
def video_images(n, seed=3):
    """n frames of a slowly changing scene at mixed sizes (each size crops / pads the same content)."""
    rs = np.random.RandomState(seed)
    base = rs.randint(0, 256, (640, 640, 3)).astype(np.int32)
    shapes = [(480, 640), (640, 480), (512, 512), (300, 400), (640, 640)]
    out = []
    for i in range(n):
        h, w = shapes[i % len(shapes)]
        img = np.clip(base + rs.randint(-5, 6, base.shape), 0, 255).astype(np.uint8)
        out.append(np.ascontiguousarray(img[:h, :w]))
    return out


@pytest.fixture(scope="module")
def romp_params():
    sd, pack = synth.romp_state_dict(0), synth.smpl_pack(0)
    frames = np.concatenate([P.img_preprocess(x, 512)[0] for x in video_images(5)])
    c, _ = O.romp_maps(sd, frames)
    sd2, _, _ = synth.calibrate_center_head(sd, c.numpy(), max_per_frame=6)
    return sd2, pack


def make(params, precision, max_batch, largest=False, smpl=True, temporal=True):
    flags = ["--precision", precision, "--max_batch", str(max_batch)]
    flags += (["-t"] + (["--show_largest"] if largest else [])) if temporal else []
    flags += [] if smpl else ["--calc_smpl"]
    return ROMP(romp_settings(flags), state_dict=params[0], smpl_pack=params[1])


TOL = dict(smpl_thetas=1e-6, smpl_betas=1e-6, cam=1e-6, cam_trans=1e-6, global_orient=1e-6, body_pose=1e-6, center_confs=1e-6,
           verts=1e-5, joints=1e-5, pj2d_org=1e-3)


def compare(got, ref, where, worst):
    assert (got is None) == (ref is None), where
    if ref is None:
        return
    assert set(got) == set(ref), (where, set(got) ^ set(ref))
    for k in ref:
        assert got[k].shape == ref[k].shape and got[k].dtype == ref[k].dtype, (where, k, got[k].shape, ref[k].shape)
        if k in ("track_ids", "center_preds"):
            assert np.array_equal(got[k], ref[k]), (where, k)
        else:
            e = float(np.abs(got[k].astype(np.float64) - ref[k]).max()) if got[k].size else 0.0
            worst[k] = max(worst.get(k, 0.0), e)
            assert e <= TOL[k], (where, k, e)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("largest", [False, True])
@pytest.mark.parametrize("smpl", [True, False])
def test_forward_video_equals_forward_loop(romp_params, precision, largest, smpl):
    imgs = video_images(11)
    sids = [0, 0, 1, 0, 1, 1, 0, 2, 0, 0, 1]
    ref_m = make(romp_params, precision, 4, largest, smpl)
    ref = [ref_m.forward(img, s) for img, s in zip(imgs, sids)]
    m = make(romp_params, precision, 4, largest, smpl)
    got = m.forward_video(imgs, sids)
    assert len(got) == len(imgs) and sum(r is not None for r in ref) >= 8
    worst = {}
    for i in range(len(imgs)):
        compare(got[i], ref[i], f"frame {i}", worst)
        if ref[i] is not None and largest:
            assert got[i]["smpl_thetas"].shape == (1, 72) and "track_ids" not in got[i]
    print(f"{precision} largest={largest} smpl={smpl}: max |forward_video - forward| " +
          ", ".join(f"{k} {v:.1e}" for k, v in sorted(worst.items())))
    # device results (to_numpy=False) carry the same values
    m.reset_temporal()
    dev = m.forward_video([torch.from_numpy(x).cuda() for x in imgs], sids, to_numpy=False)
    for i in range(len(imgs)):
        compare(None if dev[i] is None else {k: v.cpu().numpy() for k, v in dev[i].items()}, ref[i], f"device frame {i}", worst)


@pytest.mark.parametrize("largest", [False, True])
def test_forward_video_batches_equals_forward_video(romp_params, largest):
    imgs = video_images(13, seed=4)
    lists = [imgs[:3], imgs[3:4], [], imgs[4:13]]
    sids = [[0, 1, 0], [1], [], [0, 0, 1, 2, 0, 0, 1, 0, 0]]
    a = make(romp_params, "bf16", 3, largest)
    whole = a.forward_video(imgs, sum(sids, []))
    b = make(romp_params, "bf16", 3, largest)
    parts = list(b.forward_video_batches(iter(lists), iter(sids)))
    assert [len(p) for p in parts] == [len(li) for li in lists]
    flat = sum(parts, [])
    for i in range(len(imgs)):
        assert (flat[i] is None) == (whole[i] is None)
        if whole[i] is not None:
            assert set(flat[i]) == set(whole[i])
            for k in whole[i]:
                assert np.array_equal(flat[i][k], whole[i][k]), (i, k)


def moving_centers(n_frames, seed=9):
    """Center maps with 5 people walking one cell per frame, frames 3 and 7 empty, person 4 absent from frame 5 on."""
    rs = np.random.RandomState(seed)
    maps = np.zeros((n_frames, 1, 64, 64), np.float32)
    start = np.array([[8, 8], [8, 40], [40, 8], [40, 40], [24, 24]])
    step = np.array([[1, 0], [0, 1], [-1, 0], [0, -1], [1, 1]])
    vals = np.array([0.9, 0.8, 0.7, 0.6, 0.5], np.float32)
    for t in range(n_frames):
        if t in (3, 7):
            continue
        for p in range(5):
            if p == 4 and t >= 5:
                continue
            y, x = start[p] + step[p] * t
            maps[t, 0, y, x] = vals[p] + np.float32(rs.uniform(0, 0.01))
    return maps


@pytest.mark.parametrize("largest", [False, True])
def test_forward_video_planted_people_against_oracle(romp_params, largest):
    n = 12
    imgs = video_images(n, seed=6)
    maps = torch.from_numpy(moving_centers(n)).cuda()
    m = make(romp_params, "fp32", 5, largest)
    got = m.forward_video(imgs, center_override=maps)
    plain = make(romp_params, "fp32", 5, temporal=False).forward_images(imgs, center_override=maps)
    assert got[3] is None and got[7] is None and plain[3] is None
    ts, filters = TemporalState(largest), {}
    err = 0.0
    for t in range(n):
        p = plain[t]
        if p is None:
            assert got[t] is None
            continue
        g = got[t]
        slots, ids, reset = ts.assign(p["cam"], 0)
        for sl in reset:
            filters.pop(int(sl), None)
        th, be, ca = p["smpl_thetas"].copy(), p["smpl_betas"].copy(), p["cam"].copy()
        if largest:
            k = int(np.argmax(p["cam"][:, 0]))
            f = filters.setdefault(int(slots[k]), TO.make_filters(3.0))
            th, be, ca = (x[None] for x in TO.smooth(f, th[k], be[k], ca[k]))
            assert "track_ids" not in g
        else:
            for r in range(len(slots)):
                if slots[r] >= 0:
                    TO.smooth_tracked(filters.setdefault(int(slots[r]), TO.make_filters(3.0)), th[r], be[r], ca[r])
            assert np.array_equal(g["track_ids"], ids)
        assert np.array_equal(g["global_orient"], p["smpl_thetas"][:, :3]) and np.array_equal(g["center_preds"], p["center_preds"])
        assert np.abs(g["smpl_thetas"][:, :3] - th[:, :3]).max() < 1e-4
        err = max(err, float(np.abs(g["smpl_thetas"][:, 3:] - th[:, 3:]).max()), float(np.abs(g["smpl_betas"] - be).max()),
                  float(np.abs(g["cam"] - ca).max()))
    print(f"largest={largest}: max |forward_video - oracle recurrences| = {err:.2e}")
    assert err < 3e-5


def test_video_api_rules(romp_params):
    imgs = video_images(4, seed=8)
    with pytest.raises(RuntimeError):
        make(romp_params, "bf16", 2, temporal=False).forward_video(imgs)
    m = make(romp_params, "bf16", 2)
    first = m.forward_video(imgs)
    again = m.forward_video(imgs)                   # the same video goes on: ids carry over
    assert next(r for r in again if r is not None)["track_ids"].min() >= 1
    with pytest.raises(RuntimeError):
        m.forward(imgs[0])                          # forward and forward_video hold separate tracker state
    m.reset_temporal()
    restart = m.forward_video(imgs)                 # a new video: ids from 1, the same results as the first run
    for a, b in zip(first, restart):
        assert (a is None) == (b is None)
        if a is not None:
            for k in a:
                assert np.array_equal(a[k], b[k]), k
    assert min(int(r["track_ids"].min()) for r in restart if r is not None) == 1
    m.reset_temporal()
    assert m.forward(imgs[0]) is not None           # after a reset forward may take over
    with pytest.raises(RuntimeError):
        m.forward_video(imgs)
    m.reset_temporal()
    with pytest.raises(ValueError):
        m.forward_video(imgs, signal_IDs=[0, 1])
    with pytest.raises(NotImplementedError):
        m.forward_images(imgs)
