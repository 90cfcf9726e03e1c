"""Stream mode of the video paths (--video_streams): every signal_ID an independent video, all stepped by one launch.

1. BEV's track stage on a streams handle (C ABI): interleaved synthetic sequences, each stream against the oracle run on
   it alone and bit-equal to a default handle fed it alone; tracked and --show_largest; batch sizes 1, 7 and 64.
2. BEV failure isolation: a full track table fails only its stream, which works again after its reset.
3. ROMP's track stage on a streams handle: each stream bit-equal to a default handle fed it alone as signal 0, including
   100 streams cycled through batches of 64.
4. / 5. BEV and ROMP end to end: each stream equals a fresh default instance running it alone.
6. The API rules: the stream limit, reset_temporal(signal_ID), the settings checks."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import track_oracle as TO
from romp_b200 import ROMP, _lib, romp_settings, synth
from romp_b200.bev import BEV, bev_settings
from tests.test_gpu_bev_temporal import Stage, compare, moving_volumes, oracle_run
from tests.test_gpu_romp_video import add_params, cam_of, device_path, moving_centers, stage_sequence, video_images

pytestmark = pytest.mark.gpu
P = lambda t: C.c_void_p(t.data_ptr())


def interleave(lengths, mode, seed=0, starts=None):
    """(stream, frame) pairs of len(lengths) streams in one order that keeps each stream's frames in order.
    round: tick by tick (a stream joins at starts[k]); burst: random runs of 1..6 frames of one stream."""
    rs = np.random.RandomState(seed)
    if mode == "round":
        starts = starts or [0] * len(lengths)
        return sorted(((k, t) for k, n in enumerate(lengths) for t in range(n)), key=lambda e: (starts[e[0]] + e[1], e[0]))
    nxt, out = [0] * len(lengths), []
    while any(nxt[k] < n for k, n in enumerate(lengths)):
        k = rs.choice([k for k, n in enumerate(lengths) if nxt[k] < n])
        for _ in range(rs.randint(1, 7)):
            if nxt[k] < lengths[k]:
                out.append((k, nxt[k]))
                nxt[k] += 1
    return out


def same(a, b, where):
    assert (a is None) == (b is None), where
    if a is not None:
        for k in a:
            if k != "bid":                                      # the frame index within the batch
                assert np.array_equal(a[k], b[k]), (where, k)


# ------------------------------------------------------------------------------------------------
# 1. / 2. BEV stage
# ------------------------------------------------------------------------------------------------
class StreamStage(Stage):
    """b200romp_bev_track_step on a streams handle; step(frames, stream indices)."""

    def __init__(self, streams, max_tracks=128, show_largest=False):
        self.lib = _lib.load()
        self.h = self.lib.b200romp_bev_tracker_create_streams(0, max_tracks, streams)
        assert self.h, self.lib.b200romp_last_error().decode()
        self.show_largest = show_largest


def solo(seq, batch=16, **kw):
    st, out = Stage(**kw), []
    for c0 in range(0, len(seq), batch):
        r, status = st.step(seq[c0:c0 + batch], [0] * len(seq[c0:c0 + batch]))
        out += r
    return out, status


def run_streams(seqs, order, batch, show_largest=False, max_tracks=128):
    st = StreamStage(len(seqs), max_tracks, show_largest)
    got = [[None] * len(s) for s in seqs]
    statuses = []
    for c0 in range(0, len(order), batch):
        ch = order[c0:c0 + batch]
        r, status = st.step([seqs[k][t] for k, t in ch], [k for k, _ in ch])
        statuses.append((ch, status))
        for (k, t), x in zip(ch, r):
            got[k][t] = x
    return got, statuses, st


def bev_sequences(K, T, seed0=20):
    """K synthetic videos of distinct seeds and lengths, with frames holding nobody."""
    return [TO.synthetic_video(seed0 + k, T - (k % 3) * 3, (2 + k % 5, 6 + k % 9), empty_every=5 + k % 4) for k in range(K)]


@pytest.mark.parametrize("show_largest", [False, True])
@pytest.mark.parametrize("K,T,mode,batch", [(5, 24, "round", 7), (5, 24, "burst", 7), (3, 20, "late", 1), (64, 8, "round", 64),
                                            (12, 16, "burst", 64)])
def test_bev_stage_streams_equal_solo_runs(K, T, mode, batch, show_largest):
    seqs = bev_sequences(K, T)
    order = interleave([len(s) for s in seqs], "burst" if mode == "burst" else "round", seed=K,
                       starts=[(k * 5) % 11 for k in range(K)] if mode == "late" else None)
    got, statuses, _ = run_streams(seqs, order, batch, show_largest)
    assert all(s[0] == 0 for _, s in statuses)
    for k, seq in enumerate(seqs):
        ref, _ = solo(seq, show_largest=show_largest)
        for t in range(len(seq)):
            same(got[k][t], ref[t], f"stream {k} frame {t}")
        if k < 6:                                               # the oracle on the stream alone
            oref, sm = oracle_run(seq, [0] * len(seq), show_largest)
            if show_largest or sm.tracker.min_margin() > 1e-6:  # no decision of the stream near a tie
                compare(got[k], oref, f"stream {k}")


def test_bev_stage_failure_isolation_and_stream_reset():
    seqs = [TO.synthetic_video(12, 12, (56, 70))] + bev_sequences(3, 12, seed0=40)     # stream 0 overflows 8 tracks
    order = interleave([len(s) for s in seqs], "round")
    got, statuses, st = run_streams(seqs, order, 8, max_tracks=8)
    failed = [(k, t) for ch, s in statuses for (k, t), v in zip(ch, s[2:]) if v < 0]
    assert failed and {k for k, _ in failed} == {0}
    assert any(s[0] > 0 for _, s in statuses)
    first = min(t for _, t in failed)
    assert sorted(t for _, t in failed) == list(range(first, len(seqs[0])))     # stays failed until reset
    for k in (1, 2, 3):
        ref, _ = solo(seqs[k], max_tracks=8)
        for t in range(len(seqs[k])):
            same(got[k][t], ref[t], f"stream {k} frame {t}")
    st.reset(0)
    fresh = TO.synthetic_video(10, 12, (3, 4))
    r, status = st.step(fresh + seqs[1][:3], [0] * len(fresh) + [1] * 3)
    assert status[0] == 0
    ref, _ = solo(fresh, max_tracks=8)
    for t in range(len(fresh)):
        same(r[t], ref[t], f"after reset, frame {t}")


# ------------------------------------------------------------------------------------------------
# 3. ROMP stage
# ------------------------------------------------------------------------------------------------
def romp_streams_path(frames, order, largest, batch, streams):
    """b200romp_romp_track_step on a streams handle; frames[k][t] = (cam, thetas, betas, _); returns got[k][t]."""
    lib, st = _lib.load(), C.c_void_p(torch.cuda.current_stream().cuda_stream)
    h = lib.b200romp_romp_tracker_create_streams(0, streams)
    assert h
    cap = batch * 64
    z = lambda *s, dt=torch.float32: torch.zeros(*s, dtype=dt, device="cuda")
    o = dict(count=z(1, dt=torch.int32), ids=z(cap, dt=torch.int64), thetas=z(cap, 72), betas=z(cap, 10), cam=z(cap, 3),
             slot=z(cap, dt=torch.int32), track=z(cap, dt=torch.int32))
    cam, th, be, ids = z(cap, 3), z(cap, 72), z(cap, 10), z(cap, dt=torch.int64)
    got = [[None] * len(f) for f in frames]
    for c0 in range(0, len(order), batch):
        ch = [(k, t, frames[k][t]) for k, t in order[c0:c0 + batch]]
        B, ns = len(ch), [len(f[2][0]) for f in ch]
        N = sum(ns)
        cat = lambda i, w: torch.from_numpy(np.concatenate([f[2][i] for f in ch]).reshape(-1, w))
        cam[:N], th[:N], be[:N] = cat(0, 3), cat(1, 72), cat(2, 10)
        ids[:N] = torch.from_numpy(np.repeat(np.arange(B), ns).astype(np.int64))
        cnt = torch.tensor([N], dtype=torch.int32, device="cuda")
        sig = torch.tensor([k for k, _, _ in ch], dtype=torch.int32, device="cuda")
        _lib.check(lib.b200romp_romp_track_step(h, B, cap, P(cnt), P(ids), P(cam), P(th), P(be), P(sig), int(largest), 3.0, 30.0,
                                                P(o["count"]), P(o["ids"]), P(o["thetas"]), P(o["betas"]), P(o["cam"]),
                                                P(o["slot"]), P(o["track"]), st), "romp_track_step")
        torch.cuda.synchronize()
        m = int(o["count"].item())
        assert m == (sum(n > 0 for n in ns) if largest else N)
        h_ = {k: v.cpu().numpy() for k, v in o.items()}
        r0, j = 0, 0
        for b, ((k, t, _), n) in enumerate(zip(ch, ns)):
            if n == 0:
                continue
            rows = slice(j, j + 1) if largest else slice(r0, r0 + n)
            assert np.all(h_["ids"][rows] == b)
            got[k][t] = dict(slot=h_["slot"][r0:r0 + n].copy(), ids=None if largest else h_["track"][r0:r0 + n].copy(),
                             thetas=h_["thetas"][rows].copy(), betas=h_["betas"][rows].copy(), cam=h_["cam"][rows].copy())
            r0 += n
            j += 1
    lib.b200romp_romp_tracker_destroy(h)
    return got


def romp_stage_streams():
    """stage_sequence's signals as separate streams, plus a few random walks."""
    seq = add_params(stage_sequence())
    by = {}
    for f in seq:
        by.setdefault(f[3], []).append(f)
    return list(by.values())


def random_walk_streams(K, T, seed=1):
    rs = np.random.RandomState(seed)
    out = []
    for k in range(K):
        pos = rs.uniform(-800, 800, (rs.randint(1, 12), 2))
        fr = []
        for t in range(T):
            pos += rs.normal(0, 30, pos.shape)
            n = 0 if (t + k) % 6 == 5 else rs.randint(1, len(pos) + 1)
            c = cam_of(np.round(pos[rs.permutation(len(pos))[:n]]))
            c[:, 0] = rs.uniform(0.5, 1.5, n)
            fr.append((c, 0))
        out.append(add_params(fr, seed=100 + k))
    return out


@pytest.mark.parametrize("largest", [False, True])
@pytest.mark.parametrize("case", ["signals-round-7", "signals-burst-64", "walks-late-1", "walks100-round-64"])
def test_romp_stage_streams_equal_solo_runs(case, largest):
    what, mode, batch = case.split("-")
    streams = romp_stage_streams() if what == "signals" else random_walk_streams(100 if what == "walks100" else 6, 12)
    lengths = [len(s) for s in streams]
    order = interleave(lengths, "burst" if mode == "burst" else "round", seed=3,
                       starts=[(k * 7) % 13 for k in range(len(streams))] if mode == "late" else None)
    got = romp_streams_path(streams, order, largest, int(batch), len(streams))
    for k, s in enumerate(streams):
        ref = device_path([(c, th, be, 0) for c, th, be, _ in s], largest, 64)
        for t in range(len(s)):
            a, b = got[k][t], ref[t]
            assert (a is None) == (b is None), (k, t)
            if b is not None:
                for key in b:
                    assert (b[key] is None and a[key] is None) or np.array_equal(a[key], b[key]), (k, t, key)


# ------------------------------------------------------------------------------------------------
# 4. BEV end to end
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def bev_params():
    return synth.bev_damp_cam_offsets(synth.bev_state_dict(0)), synth.smpl_pack(0, num_betas=11), synth.smpl_pack(1)


def make_bev(params, precision, B, extra=()):
    return BEV(bev_settings(["--precision", precision, "--max_batch", str(B), *extra]), state_dict=params[0],
               smpla_pack=params[1], smil_pack=params[2])


def camera_volumes(K, T):
    """per camera k: moving_volumes shifted along x by 9 k cells, camera 1 with nobody at frames 2 and 3"""
    base = moving_volumes(T, empty=(4,))
    vols = []
    for k in range(K):
        v = np.roll(base, 9 * k, axis=3).copy()
        if k == 1:
            v[2:4] = 0.0
        vols.append(torch.from_numpy(v).cuda())
    return vols


def assert_results_equal(a, b, where):
    assert (a is None) == (b is None), where
    if b is not None:
        assert set(a) == set(b), (where, set(a) ^ set(b))
        for k in b:
            assert a[k].shape == b[k].shape and np.array_equal(a[k], b[k]), (where, k)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_bev_streams_end_to_end(bev_params, precision):
    K, T = 3, 6
    rs = np.random.RandomState(3)
    img = rs.randint(0, 256, (480, 640, 3)).astype(np.uint8)
    vols = camera_volumes(K, T)
    sids = ["cam-a", 17, ("c", 2)]
    m = make_bev(bev_params, precision, 2, ["-t", "--video_streams", str(K)])       # 3 frames per tick, chunks of 2
    got = [[] for _ in range(K)]
    for t in range(T):
        order = [2, 0, 1] if t % 2 else [0, 1, 2]
        vol = torch.cat([vols[k][t:t + 1] for k in order])
        out = m.forward_images([img] * K, center3d_override=vol, signal_IDs=[sids[k] for k in order])
        for k, r in zip(order, out):
            got[k].append(r)
    for k in range(K):
        ref = make_bev(bev_params, precision, 2, ["-t"]).forward_images([img] * T, center3d_override=vols[k])
        assert sum(r is not None for r in ref) >= 2
        for t in range(T):
            assert_results_equal(got[k][t], ref[t], f"{precision} camera {k} frame {t}")
        assert min(int(r["track_ids"].min()) for r in got[k] if r is not None) == 1     # ids per stream, from 1
    # forward_image_batches: the same frames as lists of one tick each (one override for every list: a still scene)
    m2 = make_bev(bev_params, precision, 4, ["-t", "--video_streams", str(K), "--show_largest"])
    vol0 = torch.cat([vols[k][0:1] for k in range(K)])
    lists = list(m2.forward_image_batches(iter([[img] * K] * 3), center3d_override=vol0, signal_IDs=iter([sids] * 3)))
    for k in range(K):
        ref = make_bev(bev_params, precision, 4, ["-t", "--show_largest"]).forward_images([img] * 3, center3d_override=vol0[k:k + 1].expand(3, -1, -1, -1).contiguous())
        for t in range(3):
            assert_results_equal(lists[t][k], ref[t], f"{precision} largest camera {k} frame {t}")


# ------------------------------------------------------------------------------------------------
# 5. ROMP end to end
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def romp_params():
    from oracle import preproc_oracle as PO
    from oracle import romp_oracle as O
    sd, pack = synth.romp_state_dict(0), synth.smpl_pack(0)
    frames = np.concatenate([PO.img_preprocess(x, 512)[0] for x in video_images(5)])
    c, _ = O.romp_maps(sd, frames)
    sd2, _, _ = synth.calibrate_center_head(sd, c.numpy(), max_per_frame=6)
    return sd2, pack


def make_romp(params, max_batch, largest=False, extra=()):
    flags = ["--precision", "bf16", "--max_batch", str(max_batch), "-t"] + (["--show_largest"] if largest else []) + list(extra)
    return ROMP(romp_settings(flags), state_dict=params[0], smpl_pack=params[1])


@pytest.mark.parametrize("largest", [False, True])
def test_romp_streams_end_to_end(romp_params, largest):
    K, T = 3, 6
    cams = [video_images(T, seed=20 + k) for k in range(K)]
    sids = [5, "b", 9]
    m = make_romp(romp_params, 2, largest, ["--video_streams", "4"])
    lists = [[cams[k][t] for k in range(K)] for t in range(T)]
    parts = list(m.forward_video_batches(iter(lists), iter([sids] * T)))
    for k in range(K):
        ref = make_romp(romp_params, 2, largest).forward_video(cams[k])
        assert sum(r is not None for r in ref) >= 4
        for t in range(T):
            assert_results_equal(parts[t][k], ref[t], f"largest={largest} camera {k} frame {t}")
    # forward(image, signal_ID) in stream mode == forward_video of the same interleaving
    f = make_romp(romp_params, 2, largest, ["--video_streams", "4"])
    loop = [f.forward(cams[k][t], sids[k]) for t in range(T) for k in (1, 0, 2)]
    v = make_romp(romp_params, 2, largest, ["--video_streams", "4"])
    whole = v.forward_video([cams[k][t] for t in range(T) for k in (1, 0, 2)], [sids[k] for t in range(T) for k in (1, 0, 2)])
    for i, (a, b) in enumerate(zip(loop, whole)):
        assert_results_equal(a, b, f"forward loop {i}")


def test_romp_streams_planted_centers(romp_params):
    n, K = 8, 2
    imgs = video_images(n, seed=6)
    maps = [torch.from_numpy(moving_centers(n, seed=9 + k)).cuda() for k in range(K)]
    m = make_romp(romp_params, 4, extra=["--video_streams", "2"])
    got = [[], []]
    for t in range(n):
        out = m.forward_video([imgs[t]] * K, [0, 1], center_override=torch.cat([maps[0][t:t + 1], maps[1][t:t + 1]]))
        got[0].append(out[0])
        got[1].append(out[1])
    for k in range(K):
        ref = make_romp(romp_params, 4).forward_video(imgs, center_override=maps[k])
        for t in range(n):
            assert_results_equal(got[k][t], ref[t], f"camera {k} frame {t}")


# ------------------------------------------------------------------------------------------------
# 6. API rules
# ------------------------------------------------------------------------------------------------
def test_bev_stream_limit_and_reset(bev_params):
    rs = np.random.RandomState(3)
    img = rs.randint(0, 256, (480, 640, 3)).astype(np.uint8)
    vols = camera_volumes(3, 6)
    m = make_bev(bev_params, "fp32", 4, ["-t", "--video_streams", "2"])
    ref = make_bev(bev_params, "fp32", 4, ["-t", "--video_streams", "2"])
    step = lambda inst, t, ks, sids: inst.forward_images([img] * len(ks), center3d_override=torch.cat([vols[k][t:t + 1] for k in ks]),
                                                         signal_IDs=sids)
    for inst in (m, ref):
        step(inst, 0, [0, 1], ["a", "b"])
    with pytest.raises(ValueError):                              # a 3rd live stream
        step(m, 1, [0, 2], ["a", "c"])
    for t in (1, 2):                                             # nothing of the refused batch was enqueued
        a, b = step(m, t, [0, 1], ["a", "b"]), step(ref, t, [0, 1], ["a", "b"])
        for x, y in zip(a, b):
            assert_results_equal(x, y, f"after the refused batch, tick {t}")
    m.reset_temporal("b")
    assert set(m.signals) == {"a"}
    c = step(m, 3, [2], ["c"])[0]                                # "c" takes b's index, afresh
    m.reset_temporal("a")
    again = step(m, 5, [0], ["a"])[0]                            # (tick 4 holds nobody)
    fresh = make_bev(bev_params, "fp32", 4, ["-t"])
    assert_results_equal(again, fresh.forward_images([img], center3d_override=vols[0][5:6])[0], "a after its reset")
    assert int(again["track_ids"].min()) == 1 and int(c["track_ids"].min()) == 1
    with pytest.raises(ValueError):
        make_bev(bev_params, "fp32", 1, ["-t"]).reset_temporal("a")
    with pytest.raises(ValueError):
        make_bev(bev_params, "fp32", 1, ["--video_streams", "2"])
    with pytest.raises(ValueError):
        make_bev(bev_params, "fp32", 1, ["-t", "--video_streams", "1025"])


def test_bev_failed_stream_is_named(bev_params):
    """A full table fails only its stream: the read-back names its signal_ID; after reset_temporal(sid) it runs again."""
    m = make_bev(bev_params, "fp32", 2, ["-t", "--video_streams", "2"])
    lib = m.lib
    lib.b200romp_bev_tracker_destroy(m.trk)                      # a handle with room for one track per stream
    m.trk = lib.b200romp_bev_tracker_create_streams(0, 1, 2)
    rs = np.random.RandomState(3)
    img = rs.randint(0, 256, (480, 640, 3)).astype(np.uint8)
    vol = torch.from_numpy(moving_volumes(1, empty=())).cuda()
    empty = torch.zeros_like(vol)
    with pytest.raises(RuntimeError, match="'x'"):
        m.forward_images([img, img], center3d_override=torch.cat([vol, empty]), signal_IDs=["x", "y"])
    m.reset_temporal("x")
    assert m.forward_images([img], center3d_override=empty, signal_IDs=["x"]) == [None]


def test_romp_stream_limit_and_reset(romp_params):
    imgs = video_images(4, seed=8)
    m = make_romp(romp_params, 2, extra=["--video_streams", "2"])
    first = m.forward_video(imgs[:2], ["a", "b"])
    with pytest.raises(ValueError):
        m.forward_video(imgs[:2], ["a", "c"])
    ref = make_romp(romp_params, 2, extra=["--video_streams", "2"])
    ref.forward_video(imgs[:2], ["a", "b"])
    for x, y in zip(m.forward_video(imgs[2:], ["a", "b"]), ref.forward_video(imgs[2:], ["a", "b"])):
        assert_results_equal(x, y, "after the refused batch")
    m.reset_temporal("a")
    restart = m.forward_video(imgs[:1], ["c"])                   # "c" takes a's index, afresh
    assert_results_equal(restart[0], first[0], "a new stream on a freed index")
    assert int(restart[0]["track_ids"].min()) == 1
    with pytest.raises(ValueError):
        make_romp(romp_params, 2).reset_temporal("a")
    with pytest.raises(ValueError):
        ROMP(romp_settings(["--video_streams", "2"]), state_dict=romp_params[0], smpl_pack=romp_params[1])
