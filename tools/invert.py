"""Latent inversion from the command line, on synthetic conditions: render a target from a hidden latent with an
eval-mode generator, then recover it from another seed with `3dhumangan_b200.inversion.invert` and print the loss curve.
    python tools/invert.py [--config 420|tiny] [--space film|z] [--steps 100] [--lr 0.02] [--loss l2|charbonnier]
                           [--hierarchical] [--checkpoint generator.pth]
                           [--perceptual-weights vgg16-397923af.pth] [--perceptual-lambda 1 1 1 1] [--no-pixel-loss]
Without --checkpoint the generator is randomly initialised and its running statistics come from three train-mode forwards
(at random initialisation the eval-mode output overflows).  --perceptual-weights adds the VGG16 perceptual term
(3dhumangan_b200.perceptual) with torchvision's VGG16 weight file; --perceptual-lambda weights its four blocks."""
import argparse
import copy
import importlib
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def released_like(pkg, which, checkpoint=None, batch=1):
    """-> (eval-mode generator, config, conditions) at the sample app's setting: 420 wide, 512x256 from a 96x48 render of 32
    steps, last_back, no density noise (`which="420"`), or a small 256-wide stand-in (`which="tiny"`)."""
    gen = importlib.import_module("3dhumangan_b200.modules.generator")
    if which == "420":
        cfg = pkg.configs.extract_metadata(copy.deepcopy(pkg.configs.MAP3DBN512L), 0)
        cfg.update(gen_height=512, gen_width=256, render_height=96, render_width=48, num_steps=32)
        if checkpoint is None:
            cfg["dataset_length"] = 16
    else:
        cfg = pkg.configs.baseline_config("tiny")
        cfg.update(gen_height=32, gen_width=32, render_height=8, render_width=8, num_steps=16)
    cfg.update(last_back=True, nerf_noise=0.0)
    torch.manual_seed(0)
    G = gen.Map3DGenerator(**cfg).cuda()
    G.set_device(torch.device("cuda:0"))
    cond = {k: v.cuda() for k, v in pkg.synthetic.make_conditions(batch, seed=1).items()}
    if checkpoint is not None:
        G.load_state_dict(torch.load(checkpoint, map_location="cuda"), strict=True)
    else:
        G.train()
        with torch.no_grad():
            for _ in range(3):
                G(torch.randn(batch, cfg["latent_dim"], device="cuda"), cond, **dict(cfg, last_back=False))
    G.eval()
    return G, cfg, cond


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", choices=["420", "tiny"], default="420")
    ap.add_argument("--space", choices=["film", "z"], default="film")
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--lr", type=float, default=0.02)
    ap.add_argument("--loss", choices=["l2", "charbonnier"], default="l2")
    ap.add_argument("--hierarchical", action="store_true")
    ap.add_argument("--checkpoint")
    ap.add_argument("--seed", type=int, default=5)
    ap.add_argument("--perceptual-weights", metavar="PATH", help="torchvision's vgg16-397923af.pth: add the perceptual term")
    ap.add_argument("--perceptual-lambda", type=float, nargs=4, default=[1.0, 1.0, 1.0, 1.0])
    ap.add_argument("--no-pixel-loss", action="store_true", help="with --perceptual-weights: the perceptual term alone")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("invert: needs a CUDA device")
    pkg = importlib.import_module("3dhumangan_b200")
    inv = importlib.import_module("3dhumangan_b200.inversion")
    G, cfg, cond = released_like(pkg, args.config, args.checkpoint)
    cfg["hierarchical_sample"] = args.hierarchical
    torch.manual_seed(11)
    with torch.no_grad():
        target = G(torch.randn(1, cfg["latent_dim"], device="cuda"), cond, **cfg)["rgbs"]
    perceptual = None
    if args.perceptual_weights:
        perceptual = importlib.import_module("3dhumangan_b200.perceptual").VGGPerceptualLoss(weights=args.perceptual_weights).cuda()
    elif args.no_pixel_loss:
        raise SystemExit("invert: --no-pixel-loss needs --perceptual-weights")
    res = inv.invert(G, target, cond, space=args.space, steps=args.steps, lr=args.lr, seed=args.seed,
                     loss=None if args.no_pixel_loss else args.loss, perceptual=perceptual,
                     **dict(cfg, perceptual_lambda=args.perceptual_lambda))
    every = max(1, args.steps // 10)
    print(json.dumps({"space": args.space, "steps": args.steps, "loss_first": res["losses"][0], "loss_last": res["losses"][-1],
                      "curve": res["losses"][::every],
                      "image_rel_l2": float((res["image"] - target).norm() / target.norm())}))


if __name__ == "__main__":
    main()
