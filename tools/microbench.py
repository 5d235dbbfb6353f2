"""Device-time measurements of the rows of SURVEY.md §8a that are not the headline bench line:
discriminator forward (a14, tensor-pipe bound), bias_act / upfirdn2d (a'1, a'2, HBM bound).

    python tools/microbench.py [--batch 8] [--iters 10] > gpurun_out/micro.json

Prints one JSON object; every number is CUDA-event time on the launching stream after warm-up, inputs
larger than L2 (or an L2 flush between iterations for the small ops).  Needs an H100 and the built library.
"""
import argparse
import importlib
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def timed(fn, iters, warmup=3, flush=None):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ms = 0.0
    for _ in range(iters):
        if flush is not None:
            flush.add_(1.0)
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        torch.cuda.synchronize()
        ms += s.elapsed_time(e)
    return ms / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--size", type=int, default=512)
    ap.add_argument("--train-batch", type=int, default=4)
    args = ap.parse_args()
    pkg = importlib.import_module("3dhumangan_b200")
    abi = importlib.import_module("3dhumangan_b200.abi")
    abi.require_device()
    peaks = {"hbm_gbps": 6573.8, "bf16_tflops": 1600.0, "source": "fallback"}
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        d = json.load(open(p))
        peaks = {"hbm_gbps": d["hbm_gbs"], "bf16_tflops": d["bf16_tflops"], "bf16_tflops_sustained": d.get("bf16_tflops_sustained"),
                 "source": "measured"}
    dev = torch.device("cuda:0")
    B, S = args.batch, args.size
    out = {"batch": B, "size": S, "peaks": peaks}
    flush = torch.zeros(64 << 20, device=dev)          # 256 MB > 126 MB L2

    # ---- discriminator forward (a14): 386.8 GFLOP / image at 512^2 as executed by the reference (SURVEY.md §8d)
    cfg = pkg.configs.baseline_config("C2")
    torch.manual_seed(0)
    disc = importlib.import_module("3dhumangan_b200.modules.discriminator")
    D = disc.UNetDiscriminator(**cfg).to(dev).train()
    img = torch.randn(B, 3, S, S, device=dev).clamp_(-1, 1)
    for mode in ("fp32x3", "bf16"):
        with torch.no_grad():
            ms = timed(lambda: D(img, None, 1.0, hg_precision=mode), args.iters)
        gflop = 386.8 * (S / 512.0) ** 2 * B
        passes = 3 if mode == "fp32x3" else 1
        out[f"discriminator_forward_{mode}"] = {
            "ms": ms, "images_per_s": B / ms * 1e3, "reference_equivalent_tflops": gflop / ms,
            "tensor_issued_tflops": gflop * passes / ms, "tensor_frac_issued": gflop * passes / ms / peaks["bf16_tflops"]}

    # ---- bias_act (a'1): read x + write y
    ba = importlib.import_module("3dhumangan_b200.ops.bias_act")
    x = torch.randn(B, 256, S, S // 2, device=dev)
    bias = torch.randn(256, device=dev)
    with torch.no_grad():
        ms = timed(lambda: ba.bias_act(x, bias, act="lrelu"), args.iters)
    nbytes = 2 * x.numel() * 4
    out["bias_act_lrelu"] = {"ms": ms, "bytes": nbytes, "gbps": nbytes / ms / 1e6, "hbm_frac": nbytes / ms / 1e6 / peaks["hbm_gbps"],
                             "shape": list(x.shape)}
    y = ba.bias_act(x.requires_grad_(False), bias, act="lrelu")
    dy = torch.randn_like(y)
    ms = timed(lambda: ba._launch_grad(dy, None, None, y, None, 1, 1, (3, 0.2, 2 ** 0.5, -1.0)), args.iters)
    nbytes = 3 * x.numel() * 4
    out["bias_act_lrelu_grad"] = {"ms": ms, "bytes": nbytes, "gbps": nbytes / ms / 1e6, "hbm_frac": nbytes / ms / 1e6 / peaks["hbm_gbps"]}
    del x, y, dy

    # ---- upfirdn2d (a'2): the reference's two call shapes (augment.py:314,325): sym6 12-tap separable, up 2 / down 2
    uf = importlib.import_module("3dhumangan_b200.ops.upfirdn2d")
    sym6 = [0.015404109327027373, 0.0034907120842174702, -0.11799011114819057, -0.048311742585633, 0.4910559419267466,
            0.787641141030194]
    f = uf.setup_filter(sym6 + sym6[::-1]).to(dev)
    xi = torch.randn(B * 8, 3, S, S, device=dev)
    with torch.no_grad():
        ms_up = timed(lambda: uf.upsample2d(xi, f, up=2), args.iters)
        up = uf.upsample2d(xi, f, up=2)
        ms_dn = timed(lambda: uf.downsample2d(up, f, down=2, padding=-6, flip_filter=True), args.iters)
        dn = uf.downsample2d(up, f, down=2, padding=-6, flip_filter=True)
    # fused two-axis kernel (hg_upfirdn2d_sep2): algorithmic bytes = read the input once + write the output once
    b_up = xi.numel() * 4 + up.numel() * 4
    b_dn = up.numel() * 4 + dn.numel() * 4
    out["upfirdn2d_upsample2d_sym6"] = {"ms": ms_up, "bytes": b_up, "gbps": b_up / ms_up / 1e6, "hbm_frac": b_up / ms_up / 1e6 / peaks["hbm_gbps"],
                                        "in": list(xi.shape), "out": list(up.shape)}
    out["upfirdn2d_downsample2d_sym6"] = {"ms": ms_dn, "bytes": b_dn, "gbps": b_dn / ms_dn / 1e6, "hbm_frac": b_dn / ms_dn / 1e6 / peaks["hbm_gbps"],
                                          "in": list(up.shape), "out": list(dn.shape)}
    # ---- synthesis network, training mode: forward (keeping the half-block inputs) + backward, C2 shape
    del D, img, xi, up, dn
    torch.cuda.empty_cache()
    st = importlib.import_module("3dhumangan_b200.modules.synthesis_train")
    gen = importlib.import_module("3dhumangan_b200.modules.generator")
    cfg = pkg.configs.baseline_config("C2")
    cfg.update(gen_height=S, gen_width=S)
    G = gen.Map3DGenerator(**cfg).to(dev).train()
    P = {k: v for k, v in list(G.named_parameters()) + list(G.named_buffers()) if k.startswith(("synthesis_network.", "synthesis_input."))}
    Rh, Rw = cfg["render_height"], cfg["render_width"]
    feat = torch.randn(B, Rh * Rw, 256, device=dev)
    fs = torch.randn(B, 256, device=dev) * 0.5
    drgb = torch.randn(B, 3, S, S, device=dev)

    def step():
        rgb, tape = st.synthesis_forward_train(P, feat, fs, cfg)
        st.synthesis_backward(P, tape, drgb)
        for p_ in P.values():
            p_.grad = None

    def fwd_only():
        st.synthesis_forward_train(P, feat, fs, cfg)

    abi.TIMING = None
    ms_f = timed(fwd_only, 3, warmup=2)
    ms_fb = timed(step, 3, warmup=2)
    torch.cuda.synchronize()
    abi.TIMING = []
    step()
    torch.cuda.synchronize()
    per = {}
    for name, s_, e_ in abi.TIMING:
        d = per.setdefault(name, [0.0, 0])
        d[0] += s_.elapsed_time(e_)
        d[1] += 1
    abi.TIMING = None
    out["synthesis_train_fp32x3"] = {"forward_ms": ms_f, "forward_backward_ms": ms_fb, "images_per_s_fwd_bwd": B / ms_fb * 1e3,
                                     "peak_mem_gb": torch.cuda.max_memory_allocated() / 1e9,
                                     "kernels_ms": {k: [round(v[0], 3), v[1]] for k, v in sorted(per.items(), key=lambda t: -t[1][0])}}
    # ---- one G+D training iteration (C3 shape, R1 weight 0 as in the 512 curricula), per-entry-point breakdown
    del P, feat, fs, drgb, G
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    ts = importlib.import_module("3dhumangan_b200.train_step")
    disc = importlib.import_module("3dhumangan_b200.modules.discriminator")
    cfg = pkg.configs.baseline_config("C2")
    cfg.update(gen_height=S, gen_width=S, nerf_noise=0.5)
    torch.manual_seed(0)
    G = gen.Map3DGenerator(**cfg).to(dev).train()
    G.set_device(dev)
    D = disc.UNetDiscriminator(**cfg).to(dev).train()
    og, od = ts.make_optimizers(G, D, cfg)
    Bt = args.train_batch
    cond = {k: v.to(dev) for k, v in pkg.synthetic.make_conditions(Bt, seed=1).items()}
    batch = dict(z_d=torch.randn(Bt, cfg["latent_dim"], device=dev), z_g=torch.randn(Bt, cfg["latent_dim"], device=dev), cond=cond,
                 images=torch.randn(Bt, 3, S, S, device=dev).clamp_(-1, 1), labels=torch.randint(1, cfg["label_dim"], (Bt, S, S), device=dev))

    def iteration():
        return ts.train_iteration(G, D, og, od, batch, cfg)

    ms_it = timed(iteration, 2, warmup=1)
    abi.TIMING = []
    torch.cuda.synchronize()
    iteration()
    torch.cuda.synchronize()
    per = {}
    for name, s_, e_ in abi.TIMING:
        d = per.setdefault(name, [0.0, 0])
        d[0] += s_.elapsed_time(e_)
        d[1] += 1
    abi.TIMING = None
    out["train_iteration_fp32x3"] = {"batch": Bt, "ms": ms_it, "images_per_s": Bt / ms_it * 1e3,
                                     "peak_mem_gb": torch.cuda.max_memory_allocated() / 1e9,
                                     "library_kernel_ms": sum(v[0] for v in per.values()),
                                     "kernels_ms": {k: [round(v[0], 3), v[1]] for k, v in sorted(per.items(), key=lambda t: -t[1][0])}}
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
