"""Per-layer device time of the discriminator's convolutions (inference path, B images at size x size): shape, kernel
variant, ms, reference-equivalent TFLOP/s and issued fraction of the bf16 tensor peak.  Needs an H100.
    python tools/dconv_layers.py [--batch 8] [--size 512] [--precision fp32x3]"""
import argparse
import importlib
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--size", type=int, default=512)
    ap.add_argument("--precision", default="fp32x3")
    args = ap.parse_args()
    pkg = importlib.import_module("3dhumangan_b200")
    abi = importlib.import_module("3dhumangan_b200.abi")
    disc = importlib.import_module("3dhumangan_b200.modules.discriminator")
    peak = 1691.2
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        peak = json.load(open(p))["bf16_tflops"]
    cfg = pkg.configs.baseline_config("C2")
    cfg.update(gen_height=args.size, gen_width=args.size)
    dev = torch.device("cuda:0")
    D = disc.UNetDiscriminator(**cfg).to(dev).train()
    img = torch.randn(args.batch, 3, args.size, args.size, device=dev).clamp_(-1, 1)
    passes = 3 if args.precision == "fp32x3" else 1
    rec = []
    orig = abi.conv2d

    def conv2d(x1, wimg, Cout, Nb, *, ksize, H, W, x2=None, **kw):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        out = orig(x1, wimg, Cout, Nb, ksize=ksize, H=H, W=W, x2=x2, **kw)
        e.record()
        cin = x1.shape[1] + (0 if x2 is None else x2.shape[1])
        rec.append((cin, Cout, H, W, ksize, bool(kw.get("up2")), s, e))
        return out

    abi.conv2d = conv2d
    with torch.no_grad():
        for _ in range(2):
            rec.clear()
            D(img, None, 1.0, hg_precision=args.precision)
    torch.cuda.synchronize()
    abi.conv2d = orig
    tot = 0.0
    rows = []
    for cin, cout, H, W, k, up2, s, e in rec:
        ms = s.elapsed_time(e)
        fl = 2.0 * args.batch * H * W * cin * cout * k * k
        halo = k == 3 and W % 128 == 0 and cin % 64 == 0 and cout <= 256 and os.environ.get("HG3D_CONV_HALO", "1") != "0"
        rows.append({"cin": cin, "cout": cout, "H": H, "W": W, "k": k, "up2": up2, "kernel": "halo" if halo else "v1", "ms": round(ms, 4),
                     "tflops_equiv": round(fl / ms / 1e9, 1), "tensor_frac_issued": round(fl * passes / ms / 1e9 / peak, 3)})
        tot += ms
    print(json.dumps({"batch": args.batch, "size": args.size, "precision": args.precision, "conv_ms_total": round(tot, 3), "layers": rows}))


if __name__ == "__main__":
    main()
