"""CPU, world_size-2 gloo: the multi-rank host logic of B200CorrespondenceGenerator for the detectors whose descriptors are not
SuperPoint's - the padded slot layout and the feature all-gather carry u8 x 128 (SIFT) and u8 x 32 (ORB) descriptors and the
keypoint sizes, masks stay on the exchange path, and keypoints, descriptors and matches equal one process's.  The batched
detector engine and the two-way matcher are replaced by deterministic stand-ins (the kernels are covered by the -m gpu suite;
tests/test_generator_detectors_multigpu_gpu.py runs the real thing on two GPUs)."""
import os

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

K = 6


class _FakeFrontEnd:
    device = torch.device("cpu")
    max_keypoints = K


class _FakeEngine:
    """extract_many: keypoint records and descriptors are functions of the image content only; a mask drops the first keypoint."""

    def __init__(self, dim):
        self.dim = dim

    def extract_many(self, images, masks=None, max_keypoints=5000):
        assert len({tuple(x.shape) for x in images}) == 1, "extract_many takes images of one shape"
        masks = masks or [None] * len(images)
        out = []
        for im, m in zip(images, masks):
            n = int(im.to(torch.int64).sum()) % max_keypoints + 1
            base = float(im.to(torch.float32).mean())
            rec = torch.zeros((n, 6))
            rec[:, 0] = base + torch.arange(n)
            rec[:, 1] = 2 * base
            rec[:, 2] = 1.6 + torch.arange(n) / 8
            rec[:, 4] = base / 255.0
            desc = ((torch.arange(n)[:, None] * 7 + torch.arange(self.dim)[None] + int(base)) % 256).to(torch.uint8)
            if m is not None:
                assert m.shape == im.shape[:2]
                rec, desc = rec[1:], desc[1:]
            out.append((rec, desc, n))
        return out


class _FakeTwoWay:
    def match_batched_dev(self, pairs, ratio=None):
        assert all(a.dtype == torch.uint8 and b.dtype == torch.uint8 for a, b in pairs)
        return [torch.stack([torch.arange(min(len(a), len(b)))] * 2, 1).to(torch.int64) for a, b in pairs]


class _Img:
    def __init__(self, arr, mask=None):
        self.value_array, self.mask = arr, mask


def _job():
    rng = np.random.default_rng(5)
    imgs = [_Img(rng.integers(0, 255, (8 + i % 2, 10), dtype=np.uint8)) for i in range(7)]  # two shapes
    imgs[5].mask = np.ones((9, 10), np.uint8)
    graph = [(i, j) for i in range(7) for j in range(i + 1, min(7, i + 3))]  # 11 pairs; image 6 only as a second member
    return imgs, graph


def _run(detector):
    from gtsfm_b200.correspondence_generator import B200CorrespondenceGenerator

    gen = B200CorrespondenceGenerator(max_keypoints=K, detector=detector, matcher="twoway", ratio_test_threshold=0.8)
    gen._fe, gen._det_engine, gen._mnn = _FakeFrontEnd(), _FakeEngine(128 if detector == "sift" else 32), _FakeTwoWay()
    imgs, graph = _job()
    kps, matches = gen.generate_correspondences(None, imgs, graph)
    return gen, kps, matches


def _same_kp(a, b):
    return all(np.array_equal(getattr(a, f), getattr(b, f)) and getattr(a, f).dtype == getattr(b, f).dtype
               for f in ("coordinates", "scales", "responses"))


def _worker(rank, world, port, q):
    single = {d: _run(d) for d in ("sift", "orb")}  # before the process group exists: world = 1
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        res = []
        for d in ("sift", "orb"):
            gen, kps, matches = _run(d)
            gen1, kps1, matches1 = single[d]
            same_kp = len(kps) == 7 and all(_same_kp(a, b) for a, b in zip(kps, kps1))
            f, f1 = gen.last_device_features, gen1.last_device_features
            same_desc = sorted(f) == sorted(f1) and all(torch.equal(f[i].desc, f1[i].desc) and f[i].desc.dtype == torch.uint8
                                                       and f[i].shape == f1[i].shape for i in f1)
            same_m = sorted(matches) == sorted(matches1) and all(np.array_equal(matches[p], matches1[p]) and matches[p].dtype == np.uint32
                                                                 for p in matches1)
            res.append((bool(same_kp), bool(same_desc), bool(same_m), gen.last_detections, int(f[0].desc.shape[1])))
        q.put((rank, res))
    finally:
        dist.destroy_process_group()


def test_two_gloo_ranks_equal_one_process_u8_descriptors():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29900 + (os.getpid() % 200)
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = dict(q.get(timeout=180) for _ in procs)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    # a masked SIFT / ORB image keeps the exchange path: 7 images detected once each (4 on rank 0, 3 on rank 1)
    assert res[0] == [(True, True, True, 4, 128), (True, True, True, 4, 32)], res
    assert res[1] == [(True, True, True, 3, 128), (True, True, True, 3, 32)], res


def test_constructor_rejects_unknown_and_mismatched_choices():
    from gtsfm_b200.correspondence_generator import B200CorrespondenceGenerator

    with pytest.raises(ValueError, match="detector"):
        B200CorrespondenceGenerator(detector="kaze", matcher="twoway")
    with pytest.raises(ValueError, match="matcher"):
        B200CorrespondenceGenerator(matcher="nn")
    with pytest.raises(ValueError, match="SuperPoint features"):
        B200CorrespondenceGenerator(detector="sift", matcher="superglue")


@pytest.mark.parametrize("detector", ["sift", "orb"])
def test_mask_of_another_shape_is_rejected(detector):
    """The batched call reads an H x W mask through its pointer alone: a mask of another shape raises the plugin's ValueError
    before any detection."""
    from gtsfm_b200.correspondence_generator import B200CorrespondenceGenerator

    gen = B200CorrespondenceGenerator(max_keypoints=K, detector=detector, matcher="twoway")
    gen._fe, gen._det_engine, gen._mnn = _FakeFrontEnd(), _FakeEngine(128 if detector == "sift" else 32), _FakeTwoWay()
    imgs, graph = _job()
    imgs[5].mask = np.ones((8, 10), np.uint8)  # image 5 is 9 x 10
    with pytest.raises(ValueError, match="height and width"):
        gen.generate_correspondences(None, imgs, graph)
