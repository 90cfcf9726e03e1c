"""Host layer of the ``romp`` / ``bev`` command lines (romp_b200/cli.py), on the CPU: frame extraction and the in-memory
JPEG round trip, ResultSaver's file names and npz contents, save_video_results, the reader thread and the arguments the
command lines refuse.  The file formats are pinned to the reference's own functions (simple_romp/romp/utils.py), loaded
through the golden generator's shim packages when the reference sources are present."""
import copy
import os
import sys

import cv2
import numpy as np
import pytest

from romp_b200 import cli

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
from make_golden import REF, load_reference  # noqa: E402


@pytest.fixture(scope="module")
def ref():
    """The reference's romp.utils, imported through the shim packages; this suite's ``romp`` / ``bev`` modules are put
    back afterwards."""
    if not os.path.isdir(REF):
        pytest.skip("reference sources not present")
    saved = {k: v for k, v in sys.modules.items() if k.split(".")[0] in ("romp", "bev")}
    try:
        for k in saved:
            del sys.modules[k]
        return load_reference()["romp.utils"]
    finally:
        for k in [k for k in sys.modules if k.split(".")[0] in ("romp", "bev")]:
            del sys.modules[k]
        sys.modules.update(saved)


def write_video(path, n=40, h=120, w=160, seed=0):
    """A seeded MJPG .avi of n frames: a noisy scene with a moving square."""
    rs = np.random.RandomState(seed)
    base = rs.randint(0, 256, (h, w, 3)).astype(np.int16)
    vw = cv2.VideoWriter(path, cv2.VideoWriter_fourcc(*"MJPG"), 24, (w, h))
    assert vw.isOpened()
    for t in range(n):
        f = np.clip(base + rs.randint(-8, 9, base.shape), 0, 255).astype(np.uint8)
        f[10 + t % 60:40 + t % 60, 20 + 2 * t:50 + 2 * t] = (40 * t) % 256
        vw.write(f)
    vw.release()


def write_folder(folder, n=7, seed=1):
    rs = np.random.RandomState(seed)
    os.makedirs(folder)
    for k in rs.permutation(n):                       # written out of order: the listing is sorted
        h, w = [(48, 64), (64, 48), (50, 50)][k % 3]
        cv2.imwrite(os.path.join(folder, f"img_{k:03d}.png"), rs.randint(0, 256, (h, w, 3)).astype(np.uint8))


def read(p):
    with open(p, "rb") as f:
        return f.read()


@pytest.mark.parametrize("save", ["out", os.path.join("out", "result.mp4")])
def test_video_frames_equal_the_reference_extraction(tmp_path, ref, save):
    video = str(tmp_path / "clip.avi")
    write_video(video)
    mine, theirs = str(tmp_path / "a" / save), str(tmp_path / "b" / save)
    frames, vpath = cli.frame_source(video, mine)
    frames = list(frames)
    rpaths, rvpath = ref.collect_frame_path(video, theirs)
    assert len(frames) == 40 and len(rpaths) == 40
    assert os.path.relpath(vpath, str(tmp_path / "a")) == os.path.relpath(rvpath, str(tmp_path / "b"))
    for (p, img), rp in zip(frames, rpaths):
        assert os.path.basename(p) == os.path.basename(rp)
        assert os.path.basename(os.path.dirname(p)) == os.path.basename(os.path.dirname(rp)) == "clip_frames"
        assert read(p) == read(rp)                                     # the bytes cv2.imwrite writes
        assert np.array_equal(img, cv2.imread(p))                      # decoded from memory = read back
    paths, vpath2 = cli.collect_frame_path(video, str(tmp_path / "c" / save))
    assert [os.path.basename(p) for p in paths] == [os.path.basename(p) for p in rpaths] and vpath2.endswith(".mp4")


def test_jpeg_round_trip_equals_imwrite_imread(tmp_path):
    rs = np.random.RandomState(3)
    for h, w in [(720, 1280), (37, 53), (1, 1)]:
        img = rs.randint(0, 256, (h, w, 3)).astype(np.uint8)
        p = str(tmp_path / f"{h}x{w}.jpg")
        assert cv2.imwrite(p, img)
        data = cli.encode_jpeg(img)
        assert data.tobytes() == read(p)
        assert np.array_equal(cv2.imdecode(data, cv2.IMREAD_COLOR), cv2.imread(p))


def test_folder_frames_equal_the_reference_listing(tmp_path, ref):
    folder = str(tmp_path / "frames")
    write_folder(folder)
    frames, vpath = cli.frame_source(folder, str(tmp_path / "out"))
    frames = list(frames)
    rpaths, rvpath = ref.collect_frame_path(folder, str(tmp_path / "out"))
    assert [p for p, _ in frames] == rpaths and vpath == rvpath
    for p, img in frames:
        assert np.array_equal(img, cv2.imread(p))
    assert not os.path.exists(str(tmp_path / "out" / "frames_frames"))


def results(n, seed):
    """Seeded per-frame results like the models': frames without anybody (None), track ids, one track skipping frames."""
    rs = np.random.RandomState(seed)
    out = []
    for t in range(n):
        if t in (2, 5):
            out.append(None)
            continue
        ids = [1, 2] + ([3] if t % 3 == 0 else [])                      # track 3 skips frames
        k = len(ids)
        out.append(dict(cam=rs.randn(k, 3).astype(np.float32), smpl_thetas=rs.randn(k, 72).astype(np.float32),
                        verts=rs.randn(k, 6890, 3).astype(np.float32), center_confs=rs.rand(k).astype(np.float32),
                        track_ids=np.array(ids, np.int32)))
    return out


def frames_on_disk(folder, n, seed=4):
    rs = np.random.RandomState(seed)
    os.makedirs(folder)
    paths = []
    for t in range(n):
        p = os.path.join(folder, f"{t:08d}.jpg")
        cv2.imwrite(p, rs.randint(0, 256, (40, 56, 3)).astype(np.uint8))
        paths.append(p)
    return paths


def same_value(a, b):
    if isinstance(a, dict):
        assert isinstance(b, dict) and list(a) == list(b)
        for k in a:
            same_value(a[k], b[k])
    elif isinstance(a, list):
        assert isinstance(b, list) and len(a) == len(b)
        for x, y in zip(a, b):
            same_value(x, y)
    else:
        x, y = np.asarray(a), np.asarray(b)
        assert x.dtype == y.dtype and x.shape == y.shape and np.array_equal(x, y)


def same_tree(d1, d2):
    """Same file names; same PNG bytes; npz files with the same arrays, key by key."""
    names = sorted(os.listdir(d1))
    assert names == sorted(os.listdir(d2))
    for name in names:
        a, b = os.path.join(d1, name), os.path.join(d2, name)
        if name.endswith(".npz"):
            x, y = np.load(a, allow_pickle=True), np.load(b, allow_pickle=True)
            assert sorted(x.files) == sorted(y.files)
            for k in x.files:
                same_value(x[k][()], y[k][()])
        else:
            assert read(a) == read(b), name
    return names


@pytest.mark.parametrize("writers", [0, 4])
@pytest.mark.parametrize("prefix", [None, "_2_0.12"])
def test_video_saver_and_results_equal_the_reference(tmp_path, ref, writers, prefix):
    n = 9
    paths = frames_on_disk(str(tmp_path / "in"), n)
    outs = results(n, seed=5)
    mine, theirs = str(tmp_path / "a"), str(tmp_path / "b")
    s = cli.ResultSaver("video", mine, writers=writers)
    r = ref.ResultSaver("video", theirs)
    for p, o in zip(paths, outs):
        s(copy.deepcopy(o), p, prefix, image=cv2.imread(p) if writers else None)
        r(copy.deepcopy(o), p, prefix=prefix)
    s.close()
    assert [os.path.relpath(p, mine) for p in s.frame_save_paths] == [os.path.relpath(p, theirs) for p in r.frame_save_paths]
    names = same_tree(mine, theirs)
    stem = lambda t: f"{t:08d}" + ("" if prefix is None else f"_{prefix}")
    assert names == sorted([stem(t) + ".png" for t in range(n)] + [stem(t) + ".npz" for t in range(n) if outs[t] is not None])

    cli.save_video_results(s.frame_save_paths)
    # the reference's save_video_results needs an npz for every frame: give the frames without anybody an empty result
    # there, and drop their (empty) entries from its results afterwards
    empty = [os.path.splitext(p)[0] + ".npz" for p, o in zip(r.frame_save_paths, outs) if o is None]
    for p in empty:
        np.savez(p, results={})
    ref.save_video_results(r.frame_save_paths)
    for p in empty:
        os.remove(p)
    got = np.load(os.path.join(mine, "video_results.npz"), allow_pickle=True)
    exp = np.load(os.path.join(theirs, "video_results.npz"), allow_pickle=True)
    exp_results = {k: v for k, v in exp["results"][()].items() if v != {}}
    same_value(got["results"][()], exp_results)
    seq = got["sequence_results"][()]
    same_value(seq, exp["sequence_results"][()])
    assert [int(t) for t in seq] == [1, 2, 3] and seq[3]["frame_id"] == [0, 3, 6]


def test_video_results_without_empty_frames_equal_the_reference(tmp_path, ref):
    n = 5
    paths = frames_on_disk(str(tmp_path / "in"), n)
    outs = [o for o in results(n + 2, seed=6) if o is not None][:n]
    s, r = cli.ResultSaver("video", str(tmp_path / "a"), writers=2), ref.ResultSaver("video", str(tmp_path / "b"))
    for p, o in zip(paths, outs):
        s(copy.deepcopy(o), p)
        r(copy.deepcopy(o), p)
    s.close()
    cli.save_video_results(s.frame_save_paths)
    ref.save_video_results(r.frame_save_paths)
    same_tree(str(tmp_path / "a"), str(tmp_path / "b"))


@pytest.mark.parametrize("save", ["res", "res.jpg", os.path.join("sub", "res.png")])
def test_image_mode_names_equal_the_reference(tmp_path, ref, save):
    """``-o`` without an extension is a directory (<stem>_<prefix>.png), with one it is the file (<name>_<prefix><ext>)."""
    p = frames_on_disk(str(tmp_path / "in"), 1)[0]
    o = results(1, seed=7)[0]
    for root, saver in (("a", cli.ResultSaver), ("b", ref.ResultSaver)):
        os.makedirs(str(tmp_path / root))
        saver("image", str(tmp_path / root / save))(copy.deepcopy(o), p, prefix="0.12")
    where = save if save == "res" else os.path.dirname(save)
    names = same_tree(str(tmp_path / "a" / where), str(tmp_path / "b" / where))
    if save == "res":
        assert names == ["00000000_0.12.npz", "00000000_0.12.png"]
    else:
        stem, ext = os.path.splitext(os.path.basename(save))
        assert f"{stem}_0.12{ext}" in names and f"{stem}_0.12.npz" in names


def test_saver_names_without_the_reference(tmp_path):
    s = cli.ResultSaver("image", str(tmp_path / "x" / "out.jpg"))
    assert s.path_of("/a/b/frame.png", "0.1") == str(tmp_path / "x" / "out_0.1.jpg")
    s = cli.ResultSaver("image", str(tmp_path / "d"))
    assert s.path_of("/a/b/frame.jpg", "0.1") == str(tmp_path / "d" / "frame_0.1.png")
    s = cli.ResultSaver("video", str(tmp_path / "v.mp4"))
    assert s.path_of("/a/00000003.jpg", "_2_0.12") == str(tmp_path / "00000003__2_0.12.png")
    assert s.path_of("/a/00000003.jpg") == str(tmp_path / "00000003.png")


def test_save_video_writes_the_saved_frames(tmp_path):
    paths = frames_on_disk(str(tmp_path / "in"), 6)
    s = cli.ResultSaver("video", str(tmp_path / "out"), writers=2)
    for p in paths:
        s(None, p)
    s.save_video(str(tmp_path / "out" / "v.mp4"), frame_rate=12)
    cap = cv2.VideoCapture(str(tmp_path / "out" / "v.mp4"))
    assert int(cap.get(cv2.CAP_PROP_FRAME_COUNT)) == 6
    assert (int(cap.get(cv2.CAP_PROP_FRAME_WIDTH)), int(cap.get(cv2.CAP_PROP_FRAME_HEIGHT))) == (56, 40)
    cap.release()


def test_read_ahead_lists_and_errors():
    assert list(cli.read_ahead(iter(range(10)), 4)) == [[0, 1, 2, 3], [4, 5, 6, 7], [8, 9]]
    assert list(cli.read_ahead(iter([]), 4)) == []

    def broken():
        yield 1
        raise ValueError("bad frame")

    with pytest.raises(ValueError, match="bad frame"):
        list(cli.read_ahead(broken(), 1))
    g = cli.read_ahead(iter(range(1000)), 2)                    # a consumer that stops early stops the reader
    assert next(g) == [0, 1]
    g.close()


def test_writer_errors_reach_the_caller(tmp_path):
    s = cli.ResultSaver("video", str(tmp_path / "out"), writers=2)
    s(None, str(tmp_path / "missing.jpg"))            # no image given and none on disk: cv2.imwrite of None fails
    with pytest.raises(Exception):
        s.close()


@pytest.mark.parametrize("argv,message", [
    (["--mode", "webcam"], "video/webcam loops are outside the hot path"),
    (["--show"], "--show is outside the GPU hot path"),
    (["--render_mesh"], "--render_mesh is outside the GPU hot path"),
    (["--mode", "video", "--render_mesh"], "--render_mesh is outside the GPU hot path"),
])
def test_romp_main_refuses_before_building_a_model(argv, message):
    from romp.main import main
    with pytest.raises(NotImplementedError, match=message):
        main(argv + ["--model_path", "/nonexistent/ROMP.pkl"])


@pytest.mark.parametrize("argv,message", [
    (["--mode", "webcam"], "webcam capture is outside the hot path"),
    (["-m", "video", "--show"], r"display \(--show\) is outside the GPU hot path"),
])
def test_bev_main_refuses_before_building_a_model(argv, message):
    from bev.main import main
    with pytest.raises(NotImplementedError, match=message):
        main(argv + ["--model_path", "/nonexistent/BEV.pth"])
