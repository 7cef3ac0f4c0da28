"""GPU, 2 devices: ONE SIFT + two-way job split over two ranks (NCCL) through B200CorrespondenceGenerator - every image detected
on one rank, the u8 x 128 descriptors and keypoint sizes all-gathered, pairs sharded p mod world, two-view verification under
the matching - gives exactly the single-process results.  Skipped on machines with one GPU."""
import os

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu


def _job():
    from gtsfm_b200 import synthetic as syn
    from gtsfm_b200.gtsfm_api import Image

    frames, cal = syn.synthetic_sequence(7, 240, 320)
    graph = [(i, j) for i in range(7) for j in range(i + 1, min(7, i + 4))]  # 15 pairs
    return [Image(f) for f in frames], graph, {i: cal for i in range(7)}


def _run(device):
    from gtsfm_b200.correspondence_generator import B200CorrespondenceGenerator

    images, graph, intr = _job()
    gen = B200CorrespondenceGenerator(max_keypoints=1000, device=device, detector="sift", matcher="twoway", ratio_test_threshold=0.8)
    kps, matches = gen.generate_correspondences(None, images, graph, verify_with=(intr, 4.0))
    return gen, kps, matches


def _worker(rank, world, port, q):
    import torch.distributed as dist

    torch.cuda.set_device(rank)
    single = _run(rank) if rank == 0 else None  # before the process group exists: world = 1
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("nccl", rank=rank, world_size=world)
    try:
        gen, kps, matches = _run(rank)
        ok, why = True, ""
        if rank == 0:
            gen1, kps1, matches1 = single
            ok = len(kps) == len(kps1) and all(all(np.array_equal(getattr(a, f), getattr(b, f)) for f in ("coordinates", "scales", "responses"))
                                               for a, b in zip(kps, kps1))
            ok = ok and all(torch.equal(gen.last_device_features[i].desc.cpu(), gen1.last_device_features[i].desc.cpu()) for i in range(7))
            why += "" if ok else "keypoints or descriptors differ; "
            same = sorted(matches) == sorted(matches1) and all(np.array_equal(matches[p], matches1[p]) and matches[p].dtype == matches1[p].dtype
                                                               for p in matches1)
            ok, why = ok and same, why + ("" if same else "matches differ; ")
            tv1 = gen1.last_two_view
            tv_ok = all(np.array_equal(gen.last_two_view[p].v_corr_idxs, tv1[p].v_corr_idxs) for p in gen.last_two_view)
            ok, why = ok and tv_ok, why + ("" if tv_ok else "two-view results differ; ")
        q.put((rank, bool(ok), why, gen.last_detections, len(gen.last_two_view)))
    finally:
        dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_two_ranks_sift_twoway_equal_one_process():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 30100 + (os.getpid() % 300)
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=300) for _ in procs)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    assert [r[1] for r in res] == [True, True], res
    assert [r[3] for r in res] == [4, 3]  # 7 images: positions 0, 2, 4, 6 on rank 0; 1, 3, 5 on rank 1 - each detected once
    assert [r[4] for r in res] == [8, 7]  # 15 pairs sharded p mod 2
