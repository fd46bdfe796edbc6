"""evaluate's gather step (evaluation.gather_scores) across a real gloo process group on the CPU: three ranks over two
images, so the last rank's slice is empty; every rank gets the single-process scores in image order and the same means."""
import os
import sys

import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N_IMAGES, WORLD = 2, 3


def per_image(i):
    """Stand-in scores of image i, each metric in the dtype the metric kernels give it."""
    return {"val_psnr": torch.tensor(30.0 + 1.25 * i, dtype=torch.float32),
            "val_psnr_y": torch.tensor(31.0 + 0.5 * i, dtype=torch.float32),
            "val_ssim": torch.tensor(0.9 + 0.01 * i, dtype=torch.float64),
            "val_ssim_y": torch.tensor(0.91 + 0.02 * i, dtype=torch.float64)}


def _worker(rank, world, port, out):
    sys.path.insert(0, ROOT)
    from _pkgload import load_package

    load_package()
    from grl_image_restoration_b200 import evaluation, sharding

    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    lo, hi = sharding.shard_range(N_IMAGES, rank, world)
    names = evaluation.COLLECTIONS["restorer"]
    r = evaluation.gather_scores([per_image(i) for i in range(lo, hi)], names, lo, hi, torch.device("cpu"))
    torch.save(dict(result=r, lohi=(lo, hi)), f"{out}.{rank}")
    dist.barrier()
    dist.destroy_process_group()


def test_gather_scores_world3_gloo_with_an_empty_rank(pkg, tmp_path):
    from grl_image_restoration_b200 import evaluation

    out = str(tmp_path / "r")
    port = 31500 + os.getpid() % 2000
    mp.spawn(_worker, args=(WORLD, port, out), nprocs=WORLD, join=True)
    single = evaluation.gather_scores([per_image(i) for i in range(N_IMAGES)], evaluation.COLLECTIONS["restorer"], 0,
                                      N_IMAGES, torch.device("cpu"))
    seen_empty = False
    for rank in range(WORLD):
        r = torch.load(f"{out}.{rank}")
        seen_empty |= r["lohi"][0] == r["lohi"][1]
        for k, v in single["scores"].items():
            got = r["result"]["scores"][k]
            assert got.dtype == v.dtype == evaluation.METRIC_DTYPES[k] and torch.equal(got, v), (rank, k)
        assert r["result"]["means"] == single["means"], rank
    assert seen_empty
