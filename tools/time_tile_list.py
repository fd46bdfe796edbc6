"""CUDA-event time of tiling.forward_tile_list against the per-image tiling.forward_tile loop it replaces, on one GPU, with
the card's name and power limit.

Workloads: the released tiled evaluations (configs.RELEASED), fp16 tensor cores, seeded random weights and images (only
the shapes matter), each on lists shaped like its test sets:
  dn-Base c3 at tile 256 / overlap 32   cbsd68  8 images, half 481 x 321 and half 321 x 481 (6 tiles each)
                                        kodak24 6 images, half 768 x 512 and half 512 x 768 (12 tiles each)
                                        set12   6 images of 256 x 256 (1 tile) and 2 of 512 x 512 (9 tiles)
  jpeg-Small c3 at 288 / 36             bsds500 8 images, half 481 x 321 and half 321 x 481 (4 tiles each)
  defocus-Base at 480 / 48              dpdd    2 frames of 1680 x 1120 (12 tiles each)
Arms: `[forward_tile(m, x[None], tile, overlap)[0] for x in list]` and `forward_tile_list(m, list, tile, overlap)`, taking
turns in one process, both eager and with use_cuda_graph; median of --iters timed runs after a warm-up that also
captures every graph.  The outputs of the two arms are checked equal before anything is printed; peak allocated memory
of each arm is measured in a run of its own.

    python tools/time_tile_list.py [--iters 3] [--lists cbsd68,kodak24,set12,bsds500,dpdd]
"""
import argparse
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from _pkgload import load_package  # noqa: E402
from time_list import peak_gb  # noqa: E402
from time_metrics import alternated_ms, power_limit  # noqa: E402

CKPT = {"dn": "dn_grl_base_c3s15.ckpt", "jpeg": "jpeg_grl_small_c3q10.ckpt",
        "defocus": "db_defocus_single_pixel_grl_base.ckpt"}
LISTS = {
    "cbsd68": ("dn", [(481, 321), (321, 481)] * 4),
    "kodak24": ("dn", [(768, 512), (512, 768)] * 3),
    "set12": ("dn", [(256, 256)] * 6 + [(512, 512)] * 2),
    "bsds500": ("jpeg", [(481, 321), (321, 481)] * 4),
    "dpdd": ("defocus", [(1120, 1680)] * 2),
}


def model(pkg, ckpt):
    import grl_oracle as orc  # weights only

    *_, tile, overlap = pkg.configs.RELEASED[ckpt]
    cfg = pkg.configs.released_config(ckpt, tile)
    m = pkg.GRL(**cfg)
    m.load_state_dict(orc.synth_state_dict(cfg, 0, "init"), strict=False)
    m = m.cuda().eval()
    m.set_precision("fp16")
    return m, tile, overlap


def workload(pkg, m, tile, overlap, task, name, sizes, iters):
    from grl_image_restoration_b200 import image_list, tiling

    g = torch.Generator(device="cuda").manual_seed(1)
    xs = [torch.rand(m.in_channels, h, w, device="cuda", generator=g) for h, w in sizes]
    tiles, chunks = tiling.tile_plan(m, image_list.network_sizes([tuple(x.shape) for x in xs]), tile, overlap)
    n_loop = sum(-(-n // 16) for n in [sum(1 for t in tiles if t[0] == i) for i in range(len(xs))])  # max_batch=16
    loop = lambda: [tiling.forward_tile(m, x[None], tile, overlap)[0] for x in xs]  # noqa: E731
    batched = lambda: tiling.forward_tile_list(m, xs, tile, overlap)  # noqa: E731
    for graph in (False, True):
        m.use_cuda_graph = graph
        m.reset_cuda_graphs()
        torch.cuda.empty_cache()
        a, b = loop(), batched()  # also captures every graph the timed runs replay
        if len(a) != len(b) or not all(torch.equal(u, v) for u, v in zip(a, b)):
            raise SystemExit(f"{task} {name} graph={graph}: forward_tile_list differs from the loop")
        del a, b
        mem = [peak_gb(loop), peak_gb(batched)]
        t_loop, t_list = alternated_ms([loop, batched], iters, warmup=1)
        mode = "graph" if graph else "eager"
        for arm, t, fwd, gb in (("loop", t_loop, n_loop, mem[0]), ("forward_tile_list", t_list, len(chunks), mem[1])):
            print(f"{task:7s} {name:7s} {mode:5s} {arm:17s}: {len(xs):2d} images {len(tiles):3d} tiles {t:9.1f} ms  "
                  f"{t / len(xs):8.2f} ms/image  {fwd:3d} forwards  peak {gb:5.1f} GiB")
        print(f"{task:7s} {name:7s} {mode:5s} speed-up x{t_loop / t_list:.2f}")
    m.use_cuda_graph = False
    m.reset_cuda_graphs()
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--lists", default=",".join(LISTS))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_tile_list.py times CUDA kernels: no GPU found")
    pkg = load_package()
    print(f"device: {torch.cuda.get_device_name()}  power limit: {power_limit()}")
    names = args.lists.split(",")
    with torch.no_grad():
        for task, ckpt in CKPT.items():
            todo = [n for n in names if LISTS[n][0] == task]
            if not todo:
                continue
            m, tile, overlap = model(pkg, ckpt)
            print(f"{ckpt}: tile {tile}, overlap {overlap}, pad_size {m.pad_size}, max_batch_tokens {m.max_batch_tokens}")
            for name in todo:
                workload(pkg, m, tile, overlap, task, name, LISTS[name][1], args.iters)
            del m
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
