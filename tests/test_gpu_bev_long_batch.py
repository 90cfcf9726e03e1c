"""BEV crowd mode for lists of wide images (BEV.process_long_images): the host plan, the segmented per-crop and merged
stages against the one-image entries image by image, and the whole path against process_long_image, all bit for bit."""
import os

import numpy as np
import pytest
import torch

from oracle import bev_oracle as B
from romp_b200 import synth
from romp_b200.bev import BEV, bev_settings, long_image_crop_table, long_image_plan, long_images_plan
from tests import bev_long_oracle as L

gpu = pytest.mark.gpu
KEYS = {"smpl_thetas", "smpl_betas", "cam", "cam_trans", "params_pred", "center_confs", "pred_batch_ids", "verts", "joints",
        "pj2d_org"}


# ------------------------------------------------------------------------------------------------ host plan (CPU)
def test_plan():
    shapes = [(1080, 2160), (1080, 3840), (400, 4000), (256, 512), (720, 2560), (1080, 3840), (200, 900)]
    p = long_images_plan(shapes, 0.8, 64)
    plans = [long_image_plan(h, w, 0.8) for h, w in shapes]
    counts = [len(q[1]) for q in plans]
    assert counts[:3] == [15, 22, 55]
    assert plans[1][1][-1, 1] - plans[1][1][-1, 0] == 911                 # 1080x3840: the narrow last crop
    assert p["first_crop"].tolist() == np.cumsum([0] + counts).tolist()
    for j, (pad, boxes, info) in enumerate(plans):
        s, e = p["first_crop"][j], p["first_crop"][j + 1]
        assert np.array_equal(p["boxes"][s:e], boxes) and p["boxes"].dtype == np.int32
        assert (p["image"][s:e] == j).all()
        assert p["row_base"][j] == 64 * s and p["pad_length"][j] == pad
        assert np.array_equal(p["pad_info"][j], info) and p["img_max_side"][j] == max(shapes[j])
    assert len(p["image"]) == len(p["boxes"]) == sum(counts)
    # passes: whole images in order, every image once, at most max(64, K of the first image) crops
    assert p["passes"] == [(0, 2), (2, 3), (3, 6), (6, 7)]
    for max_crops in (1, 8, 30, 64, 1000):
        passes = long_images_plan(shapes, 0.8, max_crops)["passes"]
        assert [i for i0, i1 in passes for i in range(i0, i1)] == list(range(len(shapes)))
        for i0, i1 in passes:
            total = sum(counts[i0:i1])
            assert i1 - i0 == 1 or total <= max(max_crops, counts[i0])
            assert i1 == len(shapes) or total + counts[i1] > max(max_crops, counts[i0])     # greedy: the next one did not fit
    assert long_images_plan(shapes, 0.8, 1)["passes"] == [(i, i + 1) for i in range(len(shapes))]
    assert long_images_plan([], 0.8, 64)["passes"] == []


# ------------------------------------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def params():
    return synth.bev_damp_cam_offsets(synth.bev_state_dict(0)), synth.smpl_pack(0, num_betas=11), synth.smpl_pack(1)


@pytest.fixture(scope="module")
def model(params):
    """model(precision, max_batch): one BEV per setting for the module"""
    made = {}

    def get(precision, max_batch):
        if (precision, max_batch) not in made:
            s = bev_settings(["--precision", precision, "--max_batch", str(max_batch)])
            made[precision, max_batch] = BEV(s, state_dict=params[0], smpla_pack=params[1], smil_pack=params[2])
        return made[precision, max_batch]
    yield get
    made.clear()


def same(a, b, what):
    assert (a is None) == (b is None), what
    if a is None:
        return
    assert set(a) == set(b) == KEYS, what
    for k in a:
        x = a[k].cpu().numpy() if isinstance(a[k], torch.Tensor) else a[k]
        y = b[k].cpu().numpy() if isinstance(b[k], torch.Tensor) else b[k]
        assert x.dtype == y.dtype and np.array_equal(x, y), f"{what}: {k}"


# stage level: the fixture's per-crop records on three images of different geometry; the second has nobody
STAGE_SHAPES = [(256, 512), (200, 500), (300, 700)]


def stage_records(golden_dir):
    z = np.load(os.path.join(golden_dir, "bev_long_post.npz"))
    assert (int(z["h"]), int(z["w"])) == STAGE_SHAPES[0]
    crops = []                                   # per global crop: the fixture's rows of crop c % 14 (none for image 1)
    for j, (h, w) in enumerate(STAGE_SHAPES):
        for c in range(len(long_image_plan(h, w, 0.8)[1])):
            crops.append(None if j == 1 else np.flatnonzero(z["crop_of"] == c % len(z["boxes"])))
    return z, crops


def fill_chunk(m, z, crops):
    """the records of a chunk's crops into the regressor's rows, grouped by crop like bev_parse3d leaves them"""
    rows = [(b, i) for b, sel in enumerate(crops) if sel is not None for i in sel]
    n = len(rows)
    b = m.buf
    if n:
        idx = np.array([i for _, i in rows])
        put = lambda key, v: b[key][:n].copy_(torch.from_numpy(np.ascontiguousarray(v)).cuda())
        put("betas", z["betas"][idx]); put("thetas", z["thetas"][idx]); put("cam", z["cam"][idx]); put("conf", z["conf"][idx])
        put("cam_trans", B.cam_to_trans(torch.from_numpy(z["cam"][idx])).numpy()); put("params_pred", z["params_pred"][idx])
        put("batch_ids", np.array([c for c, _ in rows], np.int64))
    b["count"][0] = n


def stage_one_image(m, z, crops, h, w):
    """the one-image entries (b200romp_bev_crop_post + b200romp_bev_long_merge) -> (accumulated rows, result)"""
    pad, boxes, info = long_image_plan(h, w, 0.8)
    m._long_buffers(len(boxes) * 64)
    tab = torch.from_numpy(long_image_crop_table(boxes, pad, h, w, 20.0)).cuda()
    fill_chunk(m, z, crops)
    torch.cuda.synchronize()
    with torch.cuda.stream(m.stream):
        m._long["count"].zero_()
        m.crop_post(len(boxes), 0, tab)
        m.long_merge(info, w)
    out = m._collect_long()
    lb = m._long
    n = int(lb["count"][0])
    assert int(lb["count"][1]) == sum(0 if c is None else len(c) for c in crops)
    return {k: lb[k][:n].cpu().numpy() for k in ("params_pred", "cam", "conf", "verts")}, out


@gpu
@pytest.mark.parametrize("cuts", [(10, 32), (5, 10, 15, 20, 25, 30, 35, 40, 45), (13, 14, 31, 32)])
def test_stages_segmented_bit_equal(model, golden_dir, cuts):
    """b200romp_bev_crop_post_images over chunks that straddle image boundaries (cut at `cuts`; (10, 32) gives a chunk
    with crops of all three images) and one b200romp_bev_long_merge_images == the one-image entries image by image."""
    m = model("fp32", 32)
    z, crops = stage_records(golden_dir)
    p = long_images_plan(STAGE_SHAPES, 0.8, 1000)
    assert p["passes"] == [(0, 3)]
    K, fc = len(p["boxes"]), p["first_crop"]
    ref = [stage_one_image(m, z, crops[fc[j]:fc[j + 1]], h, w) for j, (h, w) in enumerate(STAGE_SHAPES)]
    assert ref[1][1] is None and len(ref[0][0]["conf"]) > 16          # nobody in image 1; image 0 has more than one tile
    tab = np.concatenate([long_image_crop_table(p["boxes"][fc[j]:fc[j + 1]], p["pad_length"][j], h, w, 20.0)
                          for j, (h, w) in enumerate(STAGE_SHAPES)])
    base = p["row_base"].astype(np.int32)
    crops_tab = np.stack([p["image"], base[p["image"]]], 1).astype(np.int32)
    m._long_buffers(K * 64, 3)
    edges = [0, *cuts, K]
    if cuts == (10, 32):
        assert p["image"][10] == 0 and p["image"][31] == 2
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    with torch.cuda.stream(m.stream):
        m._long["count"].zero_()
    for s, e in zip(edges[:-1], edges[1:]):
        m.stream.synchronize()
        fill_chunk(m, z, crops[s:e])
        torch.cuda.synchronize()
        with torch.cuda.stream(m.stream):
            m.crop_post(e - s, s, dev(tab), dev(crops_tab))
    with torch.cuda.stream(m.stream):
        m.long_merge_images(dev(p["pad_info"]), dev(base), 64 * int(np.max(np.diff(fc))))
    got = m._collect_long_images(3)
    lb = m._long
    cnt = lb["count"][:6].cpu().numpy()
    for j in range(3):
        acc, out = ref[j]
        n = len(acc["conf"])
        assert cnt[2 * j] == n and cnt[2 * j + 1] == sum(0 if c is None else len(c) for c in crops[fc[j]:fc[j + 1]])
        for k, v in acc.items():              # per-crop survivors in crop order: kept ids, full-image cam, rows
            assert np.array_equal(lb[k][base[j]:base[j] + n].cpu().numpy(), v), f"image {j}: accumulated {k}"
        same(got[j], out, f"image {j}")


# whole path: seeded images with planted volumes; the golden image in the middle, nobody in the 4th
def whole_list(golden_dir):
    zm = np.load(os.path.join(golden_dir, "bev_long_model.npz"))
    gh, gw = int(zm["h"]), int(zm["w"])
    spec = [((300, 700), 11, 21), ((gh, gw), int(zm["image_seed"]), int(zm["vol_seed"])), ((256, 600), 12, 22),
            ((200, 900), 13, None), ((180, 640), 14, 24)]
    images, vols = [], []
    for (h, w), iseed, vseed in spec:
        k = len(long_image_plan(h, w, 0.8)[1])
        images.append(L.long_image(h, w, iseed))
        vols.append(np.zeros((k, 64, 128, 128), np.float32) if vseed is None else L.planted_volumes(k, vseed))
    return zm, images, vols


@gpu
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_whole_path_bit_equal(model, golden_dir, precision, capsys):
    """process_long_images on 5 images == process_long_image image by image, at max_batch 4 (one image per pass, chunks
    of 4), 16 and 32 (several images per pass, chunks across images); the passes agree with each other."""
    zm, images, vols = whole_list(golden_dir)
    v = [torch.from_numpy(x).cuda() for x in vols]
    vall = torch.cat(v)
    first = None
    for mb in (4, 16, 32):
        m = model(precision, mb)
        passes = long_images_plan([x.shape[:2] for x in images], 0.8, 2 * mb)["passes"]
        assert len(passes) == {4: 5, 16: 4, 32: 2}[mb] and max(i1 - i0 for i0, i1 in passes) == {4: 1, 16: 2, 32: 3}[mb]
        capsys.readouterr()
        got = m.process_long_images(images, center3d_override=vall)
        assert capsys.readouterr().out.count("No person detected!") == 1
        assert len(got) == 5 and got[3] is None and all(g is not None for i, g in enumerate(got) if i != 3)
        for i, x in enumerate(images):
            same(got[i], m.process_long_image(x, center3d_override=v[i]), f"{precision} max_batch {mb} image {i}")
        if first is None:
            first = got
        elif precision == "fp32":                # fp32 results do not depend on the batch composition
            for i in range(5):
                same(got[i], first[i], f"{precision} max_batch {mb} vs 4, image {i}")
    if precision == "fp32":
        k3 = sum(len(x) for x in vols[:3])
        one = m.process_long_images(images[:3], center3d_override=vall[:k3])     # one pass at max_batch 32
        for i in range(3):
            same(one[i], first[i], f"one pass vs one image per pass, image {i}")
        out = first[1]                           # test_end_to_end_fp32's tolerances against the golden model run
        assert out["center_confs"].tolist() == zm["center_confs"].tolist()
        assert np.abs(out["cam"] - zm["cam"]).max() < 2e-3
        assert np.abs(out["verts"][:, zm["vsel"]] - zm["verts_sel"]).max() < 2e-2
        assert np.abs(out["joints"] - zm["joints"]).max() < 2e-2


@gpu
def test_inputs(model, golden_dir):
    """Device images written on the caller's stream just before the call, host tensors, and row-strided views give
    what numpy arrays give; to_numpy=False returns tensors of their own."""
    _, images, vols = whole_list(golden_dir)
    m = model("fp32", 16)
    vall = torch.from_numpy(np.concatenate(vols)).cuda()
    want = m.process_long_images(images, center3d_override=vall)
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):                # the caller's current stream is `side`
        dev = []
        for x in images:
            big = torch.zeros((x.shape[0], x.shape[1] + 5, 3), dtype=torch.uint8, device="cuda")
            big[:, 2:2 + x.shape[1]] = torch.from_numpy(x).cuda()
            dev.append(big[:, 2:2 + x.shape[1]])                    # row stride 3 (w + 5)
        dev[0] = dev[0].contiguous()
        got = m.process_long_images(dev, center3d_override=vall, to_numpy=False)
        side.synchronize()
    for i in range(5):
        same(got[i], want[i], f"device image {i}")
    host = [torch.from_numpy(x) for x in images]
    host[2] = torch.from_numpy(np.pad(images[2], ((0, 0), (0, 3), (0, 0))))[:, :images[2].shape[1]]   # strided host view
    got = m.process_long_images(host, center3d_override=vall)
    for i in range(5):
        same(got[i], want[i], f"host tensor {i}")
    with pytest.raises(ValueError):
        m.process_long_images([images[0], np.zeros((300, 500, 3), np.uint8)])
    assert m.process_long_images([]) == []


@gpu
def test_forward_images_mixed(model, golden_dir):
    """forward_images / forward_image_batches on lists mixing normal and wide images: every element equals the image
    alone; with to_numpy=False the wide results of a list own their memory (a later list's wide images do not change
    them)."""
    _, wide, vols = whole_list(golden_dir)
    m = model("fp32", 4)
    vol_of = {x.shape[:2]: torch.from_numpy(v).cuda() for x, v in zip(wide, vols)}      # the wide shapes are distinct
    orig = m.process_long_images
    m.process_long_images = lambda imgs, **kw: orig(imgs, center3d_override=torch.cat([vol_of[tuple(t.shape[:2])] for t in imgs]),
                                                    **kw)
    rs = np.random.RandomState(5)
    normal = [rs.randint(0, 256, (rs.randint(200, 400), rs.randint(100, 300), 3)).astype(np.uint8) for _ in range(9)]   # w/h < 2
    lists = [[normal[0], wide[0], normal[1], normal[2], wide[1], normal[3], normal[4], normal[5], wide[3]],
             [wide[2], normal[6], wide[4], normal[7], normal[8]]]
    try:
        alone = [[m.forward_images([x])[0] for x in li] for li in lists]
        host = [m.forward_images(li) for li in lists]
        for li, got, ref in zip(lists, host, alone):
            for i in range(len(li)):
                same(got[i], ref[i], f"forward_images element {i}")
        gen = m.forward_image_batches(lists, to_numpy=False)
        dev = [next(gen), next(gen)]             # the second list's wide images run after the first list is yielded
        assert next(gen, None) is None
        for got, ref in zip(dev, host):
            for i in range(len(got)):
                same(got[i], ref[i], f"to_numpy=False element {i}")
    finally:
        del m.process_long_images
    assert [r is None for r in (host[0][1], host[0][4], host[0][8], host[1][0], host[1][2])] == [False, False, True, False, False]
