"""The GPU JPEG round trip (csrc/jpeg.cu through romp_b200.jpeg.FrameCodec) against cv2, byte for byte and pixel for
pixel, and the command lines' video extraction through it against the CPU path (``cli.frame_source``), file by file.
The contents and sizes are those tests/test_jpeg_oracle.py checks the numpy restatement on."""
import os
import types

import cv2
import numpy as np
import pytest
import torch

from romp_b200 import cli, jpeg
from romp_b200.bev import BEV, bev_settings
from romp_b200.main import ROMP, romp_settings
from tests.test_cli_multi_host import same_tree
from tests.test_gpu_cli import bev_files, release_device_memory, romp_files, write_folder, frame_images  # noqa: F401
from tests.test_gpu_cli_multi import planted
from tests.test_jpeg_oracle import SIZES, contents, video_frames

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def codec():
    c = jpeg.FrameCodec("cuda:0")
    assert c.usable, c.reason
    return c


def cv2_round_trip(img):
    data = cv2.imencode(".jpg", img)[1].tobytes()
    return data, cv2.imdecode(np.frombuffer(data, np.uint8), cv2.IMREAD_COLOR)


def check(out, frames):
    for (data, dev, host), img in zip(out, frames):
        ref, dec = cv2_round_trip(np.ascontiguousarray(img))
        assert data == ref
        assert np.array_equal(host, dec)
        assert np.array_equal(dev.cpu().numpy(), dec)


@pytest.mark.parametrize("size", SIZES, ids=[f"{h}x{w}" for h, w in SIZES])
def test_bytes_and_pixels_equal_cv2(codec, size):
    frames = list(contents(*size).values())
    out, event = codec.run(frames)
    event.synchronize()
    check(out, frames)


def test_video_frames_equal_cv2(codec, tmp_path):
    frames = video_frames(str(tmp_path / "clip.mp4"), 12, 360, 634)
    out, _ = codec.run(frames)
    torch.cuda.synchronize()
    check(out, frames)


def test_mixed_batch_equals_single_frames(codec):
    sizes = SIZES[:10] + [(360, 634), (64, 48)]
    frames = []
    for i in range(64):
        c = list(contents(*sizes[i % len(sizes)], seed=i).values())
        frames.append(c[i % len(c)])
    batch, _ = codec.run(frames)
    for f, (data, dev, host) in zip(frames, batch):
        [(d1, v1, h1)], _ = codec.run([f])
        assert data == d1 and np.array_equal(host, h1) and torch.equal(dev, v1)
    check(batch, frames)


def test_noise_within_bound_and_cv2_length(codec):
    for size in [(720, 1280), (1080, 1920), (1920, 1080)]:
        img = contents(*size)["noise"]
        [(data, _, _)], _ = codec.run([img])
        seg = len(data) - 623 - 2
        assert seg <= jpeg.frame_sizes(*size)["segment"]
        assert len(data) == len(cv2.imencode(".jpg", img)[1])


def test_probe_reports_another_quality_table():
    c = jpeg.FrameCodec("cuda:0", quality=90)
    assert not c.usable
    assert "other bytes" in c.reason


def test_strided_device_frames(codec):
    """Frames strided inside a larger tensor, produced on a side stream that is current when the codec runs: the codec
    reads them after that stream's work.  The producer is held back on the device first, so reading the frames
    without that ordering would see the tensor before it is filled."""
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        torch.cuda._sleep(200_000_000)                   # ~0.1 s of device time before the frames are written
        big = torch.randint(0, 256, (400, 700, 3), dtype=torch.uint8, device="cuda")
        views = [big[5:365, 7:641], big[1:18, 3:36], big[100:131, 600:601]]
        assert all(v.stride(0) == 3 * 700 for v in views)
        out, event = codec.run(views)
        side.wait_event(event)
        expected = [v.cpu().numpy() for v in views]
    check(out, expected)


# ---- the command lines: GPU extraction against the CPU path ----------------------------------------------------------

def write_video(path, n, h, w, seed):
    rs = np.random.RandomState(seed)
    base = rs.randint(0, 256, (h, w, 3)).astype(np.int16)
    vw = cv2.VideoWriter(path, cv2.VideoWriter_fourcc(*"mp4v"), 24, (w, h))
    assert vw.isOpened()
    for t in range(n):
        f = np.clip(base + rs.randint(-8, 9, base.shape), 0, 255).astype(np.uint8)
        f[h // 4:h // 2, (9 * t) % (w // 2):(9 * t) % (w // 2) + w // 5] = (30 * t) % 256
        vw.write(f)
    vw.release()
    return path


def romp_make(files, flags):
    base = ["--model_path", files["model"], "--smpl_path", files["smpl"], "--max_batch", "8"]
    return ROMP(romp_settings(base + flags), state_dict=files["sd"], smpl_pack=files["pack"])


def bev_make(files, flags):
    base = ["--model_path", files["model"], "--smpl_path", files["smpl"], "--smil_path", files["smil_file"], "--max_batch", "8"]
    return BEV(bev_settings(base + flags), state_dict=files["sd"], smpla_pack=files["smpla"], smil_pack=files["smil"])


def both_paths(monkeypatch, tmp_path, run):
    """run(out_dir) with the GPU extraction, then with frame_codec disabled (the CPU frame_source); the trees match."""
    run(str(tmp_path / "gpu"))
    with monkeypatch.context() as m:
        m.setattr(cli, "frame_codec", lambda model: None)
        run(str(tmp_path / "cpu"))
    same_tree(str(tmp_path / "gpu"), str(tmp_path / "cpu"))


@pytest.mark.parametrize("kind", ["romp", "bev"])
@pytest.mark.parametrize("flags", [[], ["-t"]], ids=["plain", "tracked"])
def test_video_mode_files_equal_cpu_extraction(monkeypatch, tmp_path, romp_files, bev_files, kind, flags):
    video = write_video(str(tmp_path / "clip.mp4"), 21, 360, 634, 3)
    files, make = (romp_files, romp_make) if kind == "romp" else (bev_files, bev_make)
    prefix = None if kind == "romp" else f"_2_{bev_settings([]).center_thresh}"
    maps = planted(kind, [(video, "people")], 70)[0]
    assert cli.frame_codec(make(files, flags)) is not None

    def run(out):
        args = types.SimpleNamespace(input=video, save_path=out, save_video=False, frame_rate=24)
        cli.run_video(make(files, flags), args, prefix, maps)

    both_paths(monkeypatch, tmp_path, run)
    frames = os.listdir(str(tmp_path / "gpu" / "clip_frames"))
    assert len(frames) == 21
    assert any(n.endswith(".npz") and n != "video_results.npz" for n in os.listdir(str(tmp_path / "gpu")))


def test_inputs_files_equal_cpu_extraction(monkeypatch, tmp_path, romp_files):
    d = tmp_path / "in"
    d.mkdir()
    paths = [write_video(str(d / "a.mp4"), 13, 360, 634, 4), write_video(str(d / "b.mp4"), 9, 240, 320, 5),
             os.path.dirname(write_folder(str(d / "folder"), frame_images(6, seed=6))[0])]

    def run(out):
        cli.run_inputs(romp_make(romp_files, ["-t", "--video_streams", "3"]), paths, out,
                       types.SimpleNamespace(open_inputs=3, save_video=False, frame_rate=24))

    both_paths(monkeypatch, tmp_path, run)
