"""BEV's video mode on the GPU: the tracker stage (csrc/track.cu) through the C ABI against oracle/track_oracle.py
(itself pinned to the reference's tracker by tests/test_oracle_bev_track_golden.py) on margin-checked synthetic
sequences, batching invariance and the capacity error; then BEV(-t / --show_largest) end to end."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import track_oracle as TO
from romp_b200 import _lib

pytestmark = pytest.mark.gpu
KEYS = ["smpl_thetas", "smpl_betas", "cam", "cam_trans", "params_pred", "center_confs", "pred_batch_ids"]
P = lambda t: C.c_void_p(t.data_ptr())


class Stage:
    """b200romp_bev_track_step on host sequences: frames are fed in batches of ``batch`` in order."""

    def __init__(self, max_tracks=128, max_signals=4, show_largest=False):
        self.lib = _lib.load()
        self.h = self.lib.b200romp_bev_tracker_create(0, max_tracks, max_signals)
        assert self.h, self.lib.b200romp_last_error().decode()
        self.show_largest = show_largest
        self.status = torch.zeros(2, dtype=torch.int32, device="cuda")

    def reset(self, signal=-1):
        _lib.check(self.lib.b200romp_bev_tracker_reset(self.h, signal, C.c_void_p(torch.cuda.current_stream().cuda_stream)))

    def step(self, frames, sigs):
        """frames: list of per-frame numpy dicts ({} = nobody).  Returns (per-frame result dicts or None, status)."""
        B = len(frames)
        cat = lambda k, shape, dt: torch.from_numpy(np.concatenate([f[k] for f in frames if f]).astype(dt) if any(frames)
                                                    else np.zeros(shape, dt)).cuda().contiguous()
        n = sum(len(f["cam"]) for f in frames if f)
        cap = max(n, 1)
        bid = torch.from_numpy(np.concatenate([np.full(len(f["cam"]), b, np.int64) for b, f in enumerate(frames) if f] or
                                              [np.zeros(0, np.int64)])).cuda()
        bid = torch.cat([bid, torch.zeros(cap - n, dtype=torch.int64, device="cuda")])
        inp = {k: cat(k, s, np.float32) for k, s in (("center_confs", (0,)), ("cam", (0, 3)), ("cam_trans", (0, 3)),
                                                        ("smpl_thetas", (0, 72)), ("smpl_betas", (0, 11)), ("params_pred", (0, 146)))}
        inp = {k: torch.cat([v, torch.zeros((cap - n,) + tuple(v.shape[1:]), device="cuda")]) for k, v in inp.items()}
        count = torch.tensor([n], dtype=torch.int32, device="cuda")
        sig = torch.tensor(sigs, dtype=torch.int32, device="cuda")
        R = 128 * B
        self.status = torch.zeros(2 + B, dtype=torch.int32, device="cuda")
        z = lambda *s, dt=torch.float32: torch.zeros(*s, dtype=dt, device="cuda")
        o = dict(count=z(1, dt=torch.int32), bid=z(R, dt=torch.int64), ids=z(R, dt=torch.int32), det=z(R, dt=torch.int32),
                 thetas=z(R, 72), betas=z(R, 11), cam=z(R, 3), cam_trans=z(R, 3), params=z(R, 146), conf=z(R))
        _lib.check(self.lib.b200romp_bev_track_step(
            self.h, B, cap, P(count), P(bid), P(inp["center_confs"]), P(inp["cam"]), P(inp["cam_trans"]), P(inp["smpl_thetas"]),
            P(inp["smpl_betas"]), P(inp["params_pred"]), P(sig), int(self.show_largest), 3.0, R, P(o["count"]), P(o["bid"]),
            P(o["ids"]), P(o["det"]), P(o["thetas"]), P(o["betas"]), P(o["cam"]), P(o["cam_trans"]), P(o["params"]), P(o["conf"]),
            P(self.status), C.c_void_p(torch.cuda.current_stream().cuda_stream)), "bev_track_step")
        torch.cuda.synchronize()
        m = int(o["count"].item())
        h = {k: v[:m].cpu().numpy() for k, v in o.items() if k != "count"}
        res = []
        status = self.status.cpu().numpy().tolist()
        for b in range(B):
            sel = h["bid"] == b
            assert status[0] or status[2 + b] == int(sel.sum())                # rows per frame
            res.append({k: v[sel] for k, v in h.items()} if sel.any() else None)
        return res, status

    def __del__(self):
        if getattr(self, "h", None):
            self.lib.b200romp_bev_tracker_destroy(self.h)


def run_stage(seq, sigs, batch, **kw):
    st = Stage(**kw)
    out = []
    for c0 in range(0, len(seq), batch):
        r, status = st.step(seq[c0:c0 + batch], sigs[c0:c0 + batch])
        assert status[0] == 0, status
        out += r
    return out, status


def oracle_run(seq, sigs, show_largest=False):
    sm = TO.TemporalBEV(show_largest=show_largest)
    return [sm(f, s) if f else None for f, s in zip(seq, sigs)], sm


def compare(got, ref, label):
    frames = 0
    for t, (g, r) in enumerate(zip(got, ref)):
        assert (g is None) == (r is None), f"{label} frame {t}: {g is None} vs {r is None}"
        if r is None:
            continue
        frames += 1
        if "track_ids" in r:
            np.testing.assert_array_equal(g["ids"], r["track_ids"], err_msg=f"{label} frame {t}")
            np.testing.assert_array_equal(g["det"], r["det_inds"], err_msg=f"{label} frame {t}")
        else:
            np.testing.assert_array_equal(g["det"], r["largest"], err_msg=f"{label} frame {t}")
        for k, gk in (("smpl_thetas", "thetas"), ("smpl_betas", "betas"), ("cam", "cam"), ("cam_trans", "cam_trans")):
            err = np.abs(g[gk] - r[k]).max()
            assert err < 3e-5, f"{label} frame {t} {k}: {err:.2e}"
        k = r["largest"] if "largest" in r else slice(None)      # --show_largest keeps every row of params / confs
        np.testing.assert_array_equal(g["params"], r["params_pred"][k])
        np.testing.assert_array_equal(g["conf"], r["center_confs"][k])
    return frames


SEEDS = [(10, (6, 12), 0), (11, (15, 30), 41), (12, (66, 80), 0)]


@pytest.mark.parametrize("seed,people,empty_every", SEEDS)
def test_stage_matches_oracle(seed, people, empty_every):
    seq = TO.synthetic_video(seed, 200, people, empty_every=empty_every)
    sigs = [0] * len(seq)
    ref, sm = oracle_run(seq, sigs)
    assert sm.tracker.min_margin() > 1e-6, "a decision of this sequence is near a tie"
    got, status = run_stage(seq, sigs, 32)
    n = compare(got, ref, f"seed {seed}")
    assert n >= 150 and status[1] == sm.tracker.frame_id
    if people[1] > 64:
        assert max(len(f["cam"]) for f in seq if f) == 64
    print(f"seed {seed}: {n} frames with rows, {sum(len(r['ids']) for r in got if r is not None)} rows match the oracle")


def test_stage_track_lifecycle_and_slot_reuse():
    """Separated people leaving and coming back: re-find from the lost list, removal after 60 lost frames (and the
    re-find of a track on the frame after its removal), removal of unconfirmed tracks, a re-lost removed track leaving
    the lists at once.  max_tracks 6 < the 9 tracks the sequence creates, so the run also needs freed slots."""
    seq = TO.separated_video(5, 180)
    sigs = [0] * len(seq)
    ref, sm = oracle_run(seq, sigs)
    ev = sm.tracker.events
    assert ev["aged"] >= 2 and ev["refind"] >= 1 and ev["refind_removed"] >= 1 and ev["unconfirmed_removed"] >= 2, ev
    assert ev["lost_in_removed"] >= 1 and sm.tracker.count > 6 and sm.tracker.min_margin() > 1e-6
    for batch in (7, 32):
        got, status = run_stage(seq, sigs, batch, max_tracks=6)
        assert compare(got, ref, f"lifecycle, batch {batch}") == len(seq) and status[1] == len(seq)


def test_stage_batching_is_bit_identical():
    seq = TO.synthetic_video(11, 120, (15, 30), empty_every=13)
    sigs = [t % 2 for t in range(len(seq))]
    runs = [run_stage(seq, sigs, b)[0] for b in (1, 7, 32)]
    ref, _ = oracle_run(seq, sigs)
    compare(runs[0], ref, "batch 1")
    for r in runs[1:]:
        for a, b in zip(runs[0], r):
            assert (a is None) == (b is None)
            if a is not None:
                for k in a:
                    if k != "bid":                                  # the frame index within the batch
                        assert np.array_equal(a[k], b[k]), k


def test_stage_show_largest_and_signals():
    seq = TO.synthetic_video(4, 60, (3, 6), empty_every=17)
    sigs = [t % 2 for t in range(len(seq))]
    ref, _ = oracle_run(seq, sigs, show_largest=True)
    got, _ = run_stage(seq, sigs, 8, show_largest=True)
    assert compare(got, ref, "largest") > 40


def test_stage_capacity_error_then_reset():
    seq = TO.synthetic_video(12, 20, (56, 70))
    st = Stage(max_tracks=8)
    _, status = st.step(seq[:4], [0] * 4)
    assert status[0] == 1
    _, status2 = st.step(seq[4:8], [0] * 4)                 # stays failed until a reset
    assert status2[0] == 1
    st.reset()
    small = TO.synthetic_video(10, 30, (3, 4))
    got, status = st.step(small, [0] * len(small))
    assert status[0] == 0
    ref, _ = oracle_run(small, [0] * len(small))
    compare(got, ref, "after reset")


# ------------------------------------------------------------------------------------------------
# BEV(-t) end to end on planted moving 3-D centre maps
# ------------------------------------------------------------------------------------------------
from romp_b200 import synth  # noqa: E402
from romp_b200.bev import BEV, bev_settings  # noqa: E402


@pytest.fixture(scope="module")
def bev_params():
    return synth.bev_damp_cam_offsets(synth.bev_state_dict(0)), synth.smpl_pack(0, num_betas=11), synth.smpl_pack(1)


def moving_volumes(T, empty=(6,)):
    """Five persons walking through the 3-D centre map, one of them with a score in (0.08, 0.12); frames in ``empty``
    hold nobody."""
    rs = np.random.RandomState(9)
    vol = rs.uniform(0, 0.05, size=(T, 64, 128, 128)).astype(np.float32)
    start = [(30, 30, 20, 0.9), (34, 30, 70, 0.8), (38, 90, 30, 0.7), (26, 90, 100, 0.6), (32, 60, 60, 0.1)]
    for t in range(T):
        if t in empty:
            vol[t] = 0.0
            continue
        for k, (z, y, x, v) in enumerate(start):
            vol[t, z, y + t, x + (t if k % 2 else -t) // 2 + 10] = v
    return vol


def make(params, precision, B, extra=()):
    return BEV(bev_settings(["--precision", precision, "--max_batch", str(B), *extra]), state_dict=params[0],
               smpla_pack=params[1], smil_pack=params[2])


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_bev_temporal_end_to_end(bev_params, precision):
    from oracle import bev_oracle as BO
    from tests.test_gpu_image_batch import assert_same, single_preprocess
    T = 10
    rs = np.random.RandomState(3)
    imgs = [rs.randint(0, 256, (480, 640, 3)).astype(np.uint8)] * T
    wide = rs.randint(0, 256, (256, 768, 3)).astype(np.uint8)
    vol = torch.from_numpy(moving_volumes(T)).cuda()
    sigs = [t % 2 for t in range(T)]
    m = make(bev_params, precision, 4, ["-t"])
    seq = imgs[:4] + [wide] + imgs[4:]                           # a wide crowd-mode image in the sequence
    got = m.forward_images(seq, center3d_override=vol, signal_IDs=sigs[:4] + [7] + sigs[4:])
    got = got[:4] + got[5:]
    assert got[6] is None                                        # the empty frame
    assert m.frame_id == T - 1                                   # ... and the wide image did not step the tracker
    # forward_images == forward_batch frame by frame on the GPU-preprocessed frames
    m1 = make(bev_params, precision, 1, ["-t"])
    frame, pad = single_preprocess(imgs[0])
    for t in range(T):
        ref = m1.forward_batch(torch.from_numpy(frame[None]), offsets=pad, img_max_side=640.0, center3d_override=vol[t:t + 1],
                               signal_IDs=[sigs[t]])
        assert (ref is None) == (got[t] is None), t
        if ref is not None:
            assert_same(got[t], ref, f"frame {t}")
            assert np.array_equal(got[t]["track_ids"], ref["track_ids"])
    # rows and ids == the oracle tracker fed with a plain instance's device parse outputs
    plain = make(bev_params, precision, 1)
    raw = make(bev_params, precision, 1, ["-t", "--calc_smpl"])
    sm = TO.TemporalBEV()
    for t in range(T):
        with torch.cuda.stream(plain.stream):
            plain.run_model(torch.from_numpy(frame[None]).cuda(), vol[t:t + 1])
        plain.stream.synchronize()
        n = int(plain.buf["count"].item())
        r = raw.forward_batch(torch.from_numpy(frame[None]), offsets=pad, img_max_side=640.0, center3d_override=vol[t:t + 1],
                              signal_IDs=[sigs[t]])
        if n == 0:
            assert r is None
            continue
        b = {k: plain.buf[s][:n].cpu().numpy() for k, s in (("smpl_thetas", "thetas"), ("smpl_betas", "betas"), ("cam", "cam"),
                                                              ("cam_trans", "cam_trans"), ("params_pred", "params_pred"),
                                                              ("center_confs", "conf"), ("pred_batch_ids", "batch_ids"))}
        o = sm(b, sigs[t])
        assert (o is None) == (r is None)
        if o is None:
            continue
        np.testing.assert_array_equal(r["track_ids"], o["track_ids"], err_msg=f"frame {t}")
        for k in ("smpl_thetas", "smpl_betas", "cam", "cam_trans"):
            assert np.abs(r[k] - o[k]).max() < 3e-5, (t, k)
        assert "verts" not in r
    assert sm.tracker.count == 4 and sm.tracker.min_margin() > 1e-6          # the person at 0.1 never starts a track
    # SMPL-A ran on the smoothed parameters; ids are shared across signals
    for g in got:
        if g is not None and len(g["cam"]):
            v, _ = BO.smpla_forward(bev_params[1], bev_params[2], g["smpl_betas"], g["smpl_thetas"])
            assert np.abs(g["verts"] - np.asarray(v)).max() < 1e-4
    assert set(got[0]["track_ids"].tolist()) & set(got[1]["track_ids"].tolist())


def test_bev_show_largest_ragged(bev_params):
    vol = torch.from_numpy(moving_volumes(3, empty=())).cuda()
    m = make(bev_params, "fp32", 3, ["-t", "--show_largest"])
    rs = np.random.RandomState(3)
    imgs = [rs.randint(0, 256, (480, 640, 3)).astype(np.uint8)] * 3
    for g in m.forward_images(imgs, center3d_override=vol):
        n = len(g["params_pred"])
        assert n >= 4 and g["center_confs"].shape == (n,) and g["pred_batch_ids"].shape == (n,)
        assert g["smpl_thetas"].shape == (1, 72) and g["cam"].shape == (1, 3) and g["cam_trans"].shape == (1, 3)
        assert g["verts"].shape == (1, 6890, 3) and "track_ids" not in g


def test_bev_temporal_signal_limit_and_reset_guard(bev_params):
    m = make(bev_params, "fp32", 8, ["-t"])
    assert m.frame_id == 0
    rs = np.random.RandomState(3)
    frames = torch.from_numpy(np.stack([rs.randint(0, 256, (512, 512, 3)).astype(np.uint8)] * 5))
    vol = torch.from_numpy(moving_volumes(5, empty=())).cuda()
    with pytest.raises(ValueError):                              # 5 distinct signals in one batch
        m.forward_batch(frames, offsets=[0, 512, 0, 512, 512, 512], center3d_override=vol, signal_IDs=[0, 1, 2, 3, 4])
    out = m.forward_batch(frames[:4], offsets=[0, 512, 0, 512, 512, 512], center3d_override=vol[:4], signal_IDs=[0, 1, 2, 3])
    assert out is not None and m.frame_id == 4
    m.forward_batch(frames[:2], offsets=[0, 512, 0, 512, 512, 512], center3d_override=vol[:2], signal_IDs=[4, 0])
    assert set(m.signals) == {0, 2, 3, 4}                        # signal 1 evicted, not signal 0 that this batch uses
    m.reset_temporal()
    assert m.signals == {}
    with pytest.raises(RuntimeError):
        make(bev_params, "fp32", 1).reset_temporal()
