"""The numpy restatement of OpenCV's JPEG round trip (tests/jpeg_oracle.py), which csrc/jpeg.cu is checked against, is
itself checked here against cv2: its file bytes equal ``cv2.imencode('.jpg')``, its decode of its own coefficients equals
``cv2.imdecode`` of those bytes, and the header romp_b200.jpeg composes equals the first 623 bytes cv2 writes, at frame
sizes with every kind of partial MCU and on contents that reach the coder's extremes."""
import cv2
import numpy as np
import pytest

from romp_b200 import jpeg
from tests import jpeg_oracle as J

# (1, 9) and (2, 17): one chroma row under fancy upsampling, whose rows above and below are that row itself
SIZES = [(1, 1), (1, 9), (2, 17), (7, 9), (8, 8), (15, 17), (16, 16), (17, 33), (31, 1), (31, 3), (31, 5), (480, 640),
         (720, 1280), (1080, 1920), (1920, 1080)]


def contents(h, w, seed=0):
    """name -> BGR frame: flat 0 and 255, uniform noise (long codes, many stuffed 0xFF bytes), horizontal and vertical
    gradients, saturated primaries (extreme Cb / Cr), a one-pixel checkerboard (every AC coefficient large)."""
    rng = np.random.default_rng(seed + h * 7919 + w)
    y, x = np.mgrid[0:h, 0:w]
    prim = np.array([(0, 0, 255), (0, 255, 0), (255, 0, 0), (255, 255, 0), (255, 0, 255), (0, 255, 255)], np.uint8)
    return {
        "zeros": np.zeros((h, w, 3), np.uint8),
        "full": np.full((h, w, 3), 255, np.uint8),
        "noise": rng.integers(0, 256, (h, w, 3), dtype=np.uint8),
        "hgrad": np.repeat((x * 255 // max(w - 1, 1)).astype(np.uint8)[..., None], 3, 2),
        "vgrad": np.stack([(y * 255 // max(h - 1, 1)), 255 - (y * 255 // max(h - 1, 1)), (x + y) % 256], -1).astype(np.uint8),
        "primaries": prim[((x // 5) + (y // 3)) % 6],
        "checker": np.repeat((((x + y) % 2) * 255).astype(np.uint8)[..., None], 3, 2),
    }


def video_frames(path, n, h, w, seed=0):
    """Frames of a synthetic mp4v video as VideoCapture reads them back."""
    rng = np.random.default_rng(seed)
    base = rng.integers(0, 256, (h, w, 3)).astype(np.int16)
    vw = cv2.VideoWriter(path, cv2.VideoWriter_fourcc(*"mp4v"), 24, (w, h))
    assert vw.isOpened()
    for t in range(n):
        f = np.clip(base + rng.integers(-8, 9, base.shape), 0, 255).astype(np.uint8)
        f[h // 4:h // 2, (9 * t) % (w // 2):(9 * t) % (w // 2) + w // 5] = (30 * t) % 256
        vw.write(f)
    vw.release()
    cap, out = cv2.VideoCapture(path), []
    while True:
        ok, f = cap.read()
        if not ok:
            break
        out.append(f)
    cap.release()
    assert len(out) == n
    return out


def check(img):
    ref = cv2.imencode(".jpg", img)[1].tobytes()
    coefs = J.forward(img)
    mine = jpeg.header(*img.shape[:2]) + J.entropy_segment(coefs) + b"\xff\xd9"
    assert mine == ref
    assert np.array_equal(J.decode(coefs, *img.shape[:2]), cv2.imdecode(np.frombuffer(ref, np.uint8), cv2.IMREAD_COLOR))


@pytest.mark.parametrize("size", SIZES, ids=[f"{h}x{w}" for h, w in SIZES])
def test_restatement_equals_cv2(size):
    for name, img in contents(*size).items():
        check(img)


def test_restatement_equals_cv2_on_video_frames(tmp_path):
    for img in video_frames(str(tmp_path / "clip.mp4"), 6, 360, 634):
        check(img)


@pytest.mark.parametrize("size", SIZES, ids=[f"{h}x{w}" for h, w in SIZES])
def test_header_equals_cv2(size):
    ref = cv2.imencode(".jpg", np.zeros((*size, 3), np.uint8))[1].tobytes()
    assert len(jpeg.header(*size)) == 623
    assert jpeg.header(*size) == ref[:623]


def test_noise_fits_the_worst_case_bound():
    """The worst-case segment bound of jpeg.frame_sizes holds for the longest segments the contents give."""
    for size in [(16, 16), (17, 33), (480, 640)]:
        seg = len(J.entropy_segment(J.forward(contents(*size)["noise"])))
        assert seg <= jpeg.frame_sizes(*size)["segment"]
