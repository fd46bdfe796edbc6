"""CUDA-event time of GRL.forward_list against the loop of B = 1 forwards it replaces, on one GPU, with the card's name
and power limit.

Workloads: GRL-Base x4 SR and GRL-Small x4 SR (the released test commands run SR on whole images, tile=0), fp16 tensor
cores, each on three lists of whole LR images:
  b100     100 images, half 120 x 80 and half 80 x 120 (the B100 test set at x4): one padded size, 128 x 128;
  mixed    a seeded list of 24 sizes between 96 and 250 pixels a side, spread over several padded sizes;
  uniform  32 images of 128 x 128, which need no padding (the control: batching only, no gather / crop work).
Arms: the loop `[model(x[None])[0] for x in list]` and `model.forward_list(list)`, taking turns in one process, both
eager and with use_cuda_graph; median of --iters timed runs after a warm-up that also captures every graph.  The outputs
of the two arms are checked equal before anything is printed.  Then the gather and crop calls alone on the b100 list's
first chunk: time (descriptor packing, output allocation and launch included), bytes moved, GB/s.

    python tools/time_list.py [--iters 3] [--models base,small] [--lists b100,mixed,uniform]
"""
import argparse
import os
import random
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from _pkgload import load_package  # noqa: E402
from time_metrics import alternated_ms, power_limit, time_ms  # noqa: E402


def lists(names):
    rnd = random.Random(0)
    out = {"b100": [(120, 80), (80, 120)] * 50,
           "mixed": [(rnd.randint(96, 250), rnd.randint(96, 250)) for _ in range(24)],
           "uniform": [(128, 128)] * 32}
    return {k: out[k] for k in names}


def model(pkg, variant):
    import grl_oracle as orc  # weights only

    cfg = pkg.configs.grl_config(variant, "sr", 4, 64)
    m = pkg.GRL(**cfg)
    m.load_state_dict(orc.synth_state_dict(cfg, 0, "init"), strict=False)
    m = m.cuda().eval()
    m.set_precision("fp16")
    return m


def peak_gb(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() / 2 ** 30


def workload(pkg, m, variant, name, sizes, iters):
    from grl_image_restoration_b200 import image_list

    g = torch.Generator(device="cuda").manual_seed(1)
    xs = [torch.rand(3, h, w, device="cuda", generator=g) for h, w in sizes]
    n_chunks = len(image_list.plan(image_list.network_sizes([tuple(x.shape) for x in xs]), m.pad_size,
                                   m.max_batch_tokens))
    loop = lambda: [m(x[None])[0] for x in xs]  # noqa: E731
    batched = lambda: m.forward_list(xs)  # noqa: E731
    for graph in (False, True):
        m.use_cuda_graph = graph
        m.reset_cuda_graphs()
        torch.cuda.empty_cache()
        a, b = loop(), batched()  # also captures every graph the timed runs replay
        if not all(torch.equal(u, v) for u, v in zip(a, b)) or len(a) != len(b):
            raise SystemExit(f"{variant} {name} graph={graph}: forward_list differs from the loop")
        del a, b
        mem = [peak_gb(loop), peak_gb(batched)]
        t_loop, t_list = alternated_ms([loop, batched], iters, warmup=1)
        for arm, t, fwd, gb in (("loop", t_loop, len(xs), mem[0]), ("forward_list", t_list, n_chunks, mem[1])):
            print(f"{variant:5s} {name:7s} {'graph' if graph else 'eager':5s} {arm:12s}: {len(xs):3d} images "
                  f"{t:9.1f} ms  {1e3 * len(xs) / t:7.1f} images/s  {t / len(xs):7.2f} ms/image  {fwd:3d} forwards  "
                  f"peak {gb:5.1f} GiB")
        print(f"{variant:5s} {name:7s} {'graph' if graph else 'eager':5s} speed-up x{t_loop / t_list:.2f}")
    m.use_cuda_graph = False
    m.reset_cuda_graphs()
    torch.cuda.empty_cache()


def gather_and_crop(pkg, iters):
    """The gather and crop of the b100 list's first chunk (64 images padded to 128 x 128, x4 outputs)."""
    from grl_image_restoration_b200 import capi, functional as K

    sizes = [(120, 80), (80, 120)] * 32
    g = torch.Generator(device="cuda").manual_seed(2)
    xs = [torch.rand(3, h, w, device="cuda", generator=g) for h, w in sizes]
    u8 = [torch.randint(0, 256, (h, w, 3), device="cuda", dtype=torch.uint8, generator=g) for h, w in sizes]
    y = torch.rand(len(sizes), 3, 512, 512, device="cuda", generator=g)
    crops = [(4 * h, 4 * w) for h, w in sizes]
    pix = sum(h * w for h, w in sizes)
    padded = len(sizes) * 128 * 128
    for name, fn, nbytes in (
            ("gather fp32", lambda: K.list_gather(xs, capi.IMAGE_F32, 3, 128, 128), 3 * 4 * (pix + padded)),
            ("gather uint8", lambda: K.list_gather(u8, capi.IMAGE_U8, 3, 128, 128), 3 * (pix + 4 * padded)),
            ("crop fp32", lambda: K.list_crop(y, crops), 3 * 16 * pix * (4 + 4)),
            ("crop uint8", lambda: K.list_crop(y, crops, u8=True), 3 * 16 * pix * (4 + 1))):
        t = time_ms(fn, max(iters, 20))
        print(f"call {name:12s}: {t * 1e3:8.1f} us  {nbytes / 1e6:7.2f} MB  {nbytes / (t * 1e-3) / 1e9:7.1f} GB/s  "
              f"(64 images, batch 128 x 128; descriptor packing, output allocation and launch included)")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--models", default="base,small")
    ap.add_argument("--lists", default="b100,mixed,uniform")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_list.py times CUDA kernels: no GPU found")
    pkg = load_package()
    print(f"device: {torch.cuda.get_device_name()}  power limit: {power_limit()}")
    with torch.no_grad():
        gather_and_crop(pkg, args.iters)
        for variant in args.models.split(","):
            m = model(pkg, variant)
            print(f"{variant}: pad_size {m.pad_size}, max_batch_tokens {m.max_batch_tokens}")
            for name, sizes in lists(args.lists.split(",")).items():
                workload(pkg, m, variant, name, sizes, args.iters)
            del m
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
