"""FID statistics and distances with 3dhumangan_b200.fid.

    python tools/fid.py real --images DIR --out real.npz [--batch 64] [--inception PATH]
    python tools/fid.py gen  --config 420|tiny [--checkpoint generator.pth] --num N --out gen.npz [--batch 8] [--seed 0]
                             [--truncation 1.0] [--inception PATH]
    python tools/fid.py fid  a.npz b.npz

`real` reads every PNG / JPEG under DIR with torchvision.io at its stored size (resizing a dataset to the generator's
resolution belongs to the data pipeline) and writes pytorch-fid's statistics file (`mu`, `sigma`).  `gen` samples the
generator as the sample app does, on synthetic bodies (so its FID is not comparable with the paper's SHHQ-pose numbers);
without --checkpoint the parameters are seeded.  It runs under torchrun as well: every rank renders its share and rank 0
writes the file.  `fid` prints the Frechet distance of two statistics files and needs no GPU.  --inception defaults to
pytorch-fid's cached weights, which are never downloaded."""
import argparse
import importlib
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def _fid():
    return importlib.import_module("3dhumangan_b200.fid")


def _images(folder):
    exts = (".png", ".jpg", ".jpeg")
    return sorted(os.path.join(d, f) for d, _, fs in os.walk(folder) for f in fs if f.lower().endswith(exts))


def real(args):
    import torchvision.io as tio
    fid = _fid()
    paths = _images(args.images)
    if len(paths) < 2:
        raise SystemExit(f"fid real: need at least 2 images under {args.images} (found {len(paths)})")
    net = fid.FIDInceptionV3(weights=args.inception).cuda()
    stats = fid.FeatureStats()
    batch = []

    def flush():
        # images of different sizes go through the network one size at a time
        by_size = {}
        for im in batch:
            by_size.setdefault(tuple(im.shape), []).append(im)
        for ims in by_size.values():
            stats.update(net.features(torch.stack(ims).cuda()))
        batch.clear()

    for p in paths:
        im = tio.decode_image(tio.read_file(p), mode=tio.ImageReadMode.RGB)
        batch.append(im)
        if len(batch) == args.batch:
            flush()
    if batch:
        flush()
    stats.save(args.out)
    print(f"{stats.n} images -> {args.out}")


def gen(args):
    import torch.distributed as dist
    from invert import released_like
    pkg = importlib.import_module("3dhumangan_b200")
    fid = _fid()
    if "RANK" in os.environ and not dist.is_initialized():
        torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", 0)))
        dist.init_process_group("nccl")
    G, cfg, _ = released_like(pkg, args.config, args.checkpoint)
    G.set_device(torch.device("cuda", torch.cuda.current_device()))
    net = fid.FIDInceptionV3(weights=args.inception).cuda()
    rank = dist.get_rank() if dist.is_initialized() else 0
    torch.manual_seed(args.seed + rank)              # the renderer's ray jitter
    stats = fid.generator_statistics(G, cfg, args.num, args.batch, seed=args.seed, truncation_psi=args.truncation,
                                     inception=net)
    if rank == 0:
        stats.save(args.out)
        print(f"{stats.n} images -> {args.out}")
    if dist.is_initialized():
        dist.destroy_process_group()


def distance(args):
    fid = _fid()
    print(f"{fid.frechet_distance(*fid.load_stats(args.a), *fid.load_stats(args.b)):.6f}")


def main():
    ap = argparse.ArgumentParser()
    sub = ap.add_subparsers(dest="cmd", required=True)
    r = sub.add_parser("real")
    r.add_argument("--images", required=True)
    r.add_argument("--out", required=True)
    r.add_argument("--batch", type=int, default=64)
    r.add_argument("--inception")
    g = sub.add_parser("gen")
    g.add_argument("--config", choices=["420", "tiny"], default="420")
    g.add_argument("--checkpoint")
    g.add_argument("--num", type=int, required=True)
    g.add_argument("--out", required=True)
    g.add_argument("--batch", type=int, default=8)
    g.add_argument("--seed", type=int, default=0)
    g.add_argument("--truncation", type=float, default=1.0)
    g.add_argument("--inception")
    f = sub.add_parser("fid")
    f.add_argument("a")
    f.add_argument("b")
    args = ap.parse_args()
    if args.cmd != "fid" and not torch.cuda.is_available():
        raise SystemExit(f"fid {args.cmd}: needs a CUDA device")
    {"real": real, "gen": gen, "fid": distance}[args.cmd](args)


if __name__ == "__main__":
    main()
