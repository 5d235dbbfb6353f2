"""Feature banks and every metric from them with 3dhumangan_b200.metrics: FID, KID and precision / recall.

    python tools/evaluate.py real  --images DIR --out real_feats.npz [--batch 64] [--inception PATH] [--vgg PATH]
    python tools/evaluate.py gen   --config 420|tiny [--checkpoint generator.pth] --num N --out gen_feats.npz [--batch 8]
                                   [--seed 0] [--truncation 1.0] [--inception PATH] [--vgg PATH]
    python tools/evaluate.py score real_feats.npz gen_feats.npz [--subsets 100] [--subset-size 1000] [--k 3]
    python tools/evaluate.py ppl   --config 420|tiny [--checkpoint generator.pth] [--num 50000] [--batch 8] [--seed 0]
                                   [--space w|z] [--sampling end|full] [--epsilon 1e-4] [--truncation 1.0] [--vgg PATH]
                                   [--lpips PATH]

`real` reads the image folder under the rules of `tools/fid.py real` (every PNG / JPEG at its stored size) and `gen` samples
the generator as `tools/fid.py gen` does (same seeds, same ray-jitter seeding, torchrun-capable, rank 0 writes).  Both write
one .npz with the Inception pool features (`inception`, [N,2048]) and the VGG16 fc7 features (`vgg16`, [N,4096]) of every
image, so all metrics come from one pass over the images.  `score` prints one JSON line with `fid`, `kid`, `kid_std`,
`precision`, `recall`, `n_real`, `n_gen`, `k`, `subsets` and `subset_size`.  `ppl` prints one JSON line with the perceptual
path length of the generator (`3dhumangan_b200.ppl.path_length`; torchrun-capable like `gen`, rank 0 prints): `ppl`, `lo`,
`hi`, `num`, `batch`, `seed`, `space`, `sampling`, `epsilon` and `truncation`.  The detectors' weights default to the cached
pytorch-fid and torchvision files, and LPIPS's lin weights to `ppl.default_lin_path()`; none is ever downloaded."""
import argparse
import importlib
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def _mods():
    return importlib.import_module("3dhumangan_b200.fid"), importlib.import_module("3dhumangan_b200.metrics")


def real(args):
    import torchvision.io as tio
    from fid import _images
    fid, metrics = _mods()
    paths = _images(args.images)
    if len(paths) < 2:
        raise SystemExit(f"evaluate real: need at least 2 images under {args.images} (found {len(paths)})")
    inc = fid.FIDInceptionV3(weights=args.inception).cuda()
    vgg = metrics.VGG16Features(weights=args.vgg).cuda()
    feats = {"inception": [], "vgg16": []}
    batch = []

    def flush():
        # images of different sizes go through the networks one size at a time, in file order within a size
        by_size = {}
        for im in batch:
            by_size.setdefault(tuple(im.shape), []).append(im)
        for ims in by_size.values():
            x = torch.stack(ims).cuda()
            feats["inception"].append(inc.features(x))
            feats["vgg16"].append(vgg.features(x))
        batch.clear()

    for p in paths:
        batch.append(tio.decode_image(tio.read_file(p), mode=tio.ImageReadMode.RGB))
        if len(batch) == args.batch:
            flush()
    if batch:
        flush()
    out = {k: torch.cat(v) for k, v in feats.items()}
    metrics.save_features(args.out, out)
    print(f"{out['inception'].shape[0]} images -> {args.out}")


def gen(args):
    import torch.distributed as dist
    from invert import released_like
    pkg = importlib.import_module("3dhumangan_b200")
    fid, metrics = _mods()
    if "RANK" in os.environ and not dist.is_initialized():
        torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", 0)))
        dist.init_process_group("nccl")
    G, cfg, _ = released_like(pkg, args.config, args.checkpoint)
    G.set_device(torch.device("cuda", torch.cuda.current_device()))
    inc = fid.FIDInceptionV3(weights=args.inception).cuda()
    vgg = metrics.VGG16Features(weights=args.vgg).cuda()
    rank = dist.get_rank() if dist.is_initialized() else 0
    torch.manual_seed(args.seed + rank)              # the renderer's ray jitter, seeded as tools/fid.py gen seeds it
    feats = metrics.generator_features(G, cfg, args.num, args.batch, seed=args.seed, truncation_psi=args.truncation,
                                       inception=inc, vgg=vgg)
    if rank == 0:
        metrics.save_features(args.out, feats)
        print(f"{args.num} images -> {args.out}")
    if dist.is_initialized():
        dist.destroy_process_group()


def ppl(args):
    import torch.distributed as dist
    from invert import released_like
    pkg = importlib.import_module("3dhumangan_b200")
    metrics = importlib.import_module("3dhumangan_b200.metrics")
    ppl_mod = importlib.import_module("3dhumangan_b200.ppl")
    if "RANK" in os.environ and not dist.is_initialized():
        torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", 0)))
        dist.init_process_group("nccl")
    G, cfg, _ = released_like(pkg, args.config, args.checkpoint)
    G.set_device(torch.device("cuda", torch.cuda.current_device()))
    lpips = ppl_mod.LPIPS(vgg=metrics.VGG16Features(weights=args.vgg), lin=args.lpips).cuda()
    res = ppl_mod.path_length(G, cfg, args.num, args.batch, seed=args.seed, space=args.space, sampling=args.sampling,
                              epsilon=args.epsilon, truncation_psi=args.truncation, lpips=lpips)
    if not dist.is_initialized() or dist.get_rank() == 0:
        print(json.dumps({"ppl": res["ppl"], "lo": res["lo"], "hi": res["hi"], "num": args.num, "batch": args.batch,
                          "seed": args.seed, "space": args.space, "sampling": args.sampling, "epsilon": args.epsilon,
                          "truncation": args.truncation}))
    if dist.is_initialized():
        dist.destroy_process_group()


def score(args):
    fid, metrics = _mods()
    r, g = metrics.load_features(args.real), metrics.load_features(args.gen)
    stats = []
    for f in (r, g):
        st = fid.FeatureStats()
        st.update(f["inception"].cuda())
        stats.append(st.mean_cov())
    fd = fid.frechet_distance(*stats[0], *stats[1])
    kid, kid_std, t = metrics.kid(r["inception"].cuda(), g["inception"].cuda(), args.subsets, args.subset_size)
    precision, recall = metrics.precision_recall(r["vgg16"].cuda(), g["vgg16"].cuda(), args.k)
    n_r, n_g = r["inception"].shape[0], g["inception"].shape[0]
    print(json.dumps({"fid": fd, "kid": kid, "kid_std": kid_std, "precision": precision, "recall": recall, "n_real": n_r,
                      "n_gen": n_g, "k": args.k, "subsets": len(t), "subset_size": min(n_r, n_g, args.subset_size)}))


def parser():
    ap = argparse.ArgumentParser()
    sub = ap.add_subparsers(dest="cmd", required=True)
    r = sub.add_parser("real")
    r.add_argument("--images", required=True)
    r.add_argument("--out", required=True)
    r.add_argument("--batch", type=int, default=64)
    r.add_argument("--inception")
    r.add_argument("--vgg")
    g = sub.add_parser("gen")
    g.add_argument("--config", choices=["420", "tiny"], default="420")
    g.add_argument("--checkpoint")
    g.add_argument("--num", type=int, required=True)
    g.add_argument("--out", required=True)
    g.add_argument("--batch", type=int, default=8)
    g.add_argument("--seed", type=int, default=0)
    g.add_argument("--truncation", type=float, default=1.0)
    g.add_argument("--inception")
    g.add_argument("--vgg")
    s = sub.add_parser("score")
    s.add_argument("real")
    s.add_argument("gen")
    s.add_argument("--subsets", type=int, default=100)
    s.add_argument("--subset-size", type=int, default=1000)
    s.add_argument("--k", type=int, default=3)
    p = sub.add_parser("ppl")
    p.add_argument("--config", choices=["420", "tiny"], default="420")
    p.add_argument("--checkpoint")
    p.add_argument("--num", type=int, default=50000)
    p.add_argument("--batch", type=int, default=8)
    p.add_argument("--seed", type=int, default=0)
    p.add_argument("--space", choices=["w", "z"], default="w")
    p.add_argument("--sampling", choices=["end", "full"], default="end")
    p.add_argument("--epsilon", type=float, default=1e-4)
    p.add_argument("--truncation", type=float, default=1.0)
    p.add_argument("--vgg")
    p.add_argument("--lpips")
    return ap


def main(argv=None):
    args = parser().parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit(f"evaluate {args.cmd}: needs a CUDA device")
    {"real": real, "gen": gen, "score": score, "ppl": ppl}[args.cmd](args)


if __name__ == "__main__":
    main()
