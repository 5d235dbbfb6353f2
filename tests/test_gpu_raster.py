"""The SMPL label-map rasteriser on the device (3dhumangan_b200/preprocess.py, csrc/raster.cu) against the CPU oracle
(oracle/raster_port.py, pinned to the reference's preprocessor by tests/test_oracle_pin_raster.py), the generator's camera, and
the trainer's target schedule (SURVEY.md 8f-2)."""
import importlib
import os
import random
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import raster_port as rp
from oracle import smpl_port as sp

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
sys.path.insert(0, GOLD)
import make_golden_raster as mg      # noqa: E402  (seeded conditions of the synthetic surface)


def _pre():
    return importlib.import_module("3dhumangan_b200.preprocess")


def _labels():
    return rp.faces_to_labels(os.path.join(GOLD, "densepose_data.json"))


def _body_case(B, H, W, seed):
    cond, faces, ang = mg.conditions(B, seed)
    R, T, focal = rp.camera(cond, ang[0], ang[1], ang[2])
    proj = rp.project(cond["vertices"].numpy(), R.numpy(), T.numpy(), focal)
    return cond, faces.numpy(), ang, proj, _labels().numpy(), cond["tpose_vertices"][0].numpy()


def _soup(seed=5):
    """64x64 triangle soup: large overlapping faces (warp path), small ones (thread path), coplanar copies (exact depth ties),
    zero-area and behind-camera faces."""
    g = np.random.default_rng(seed)
    tris = []
    for _ in range(120):
        tris.append(np.c_[g.uniform(-1.3, 1.3, (3, 2)), np.full(3, g.choice([1.0, 2.0, 4.0]))])
    for _ in range(300):
        c = g.uniform(-1, 1, 2)
        tris.append(np.c_[c + g.uniform(-0.08, 0.08, (3, 2)), np.full(3, g.uniform(0.5, 5))])
    for _ in range(40):
        c = g.uniform(-1, 1, 2)
        tris.append(np.c_[c + g.uniform(-0.5, 0.5, (3, 2)), g.uniform(0.5, 5, 3)])          # slanted
    tris.append(np.array([[0.0, 0.0, 1.0], [0.5, 0.5, 1.0], [1.0, 1.0, 1.0]]))              # zero area
    tris.append(np.array([[1.0, 1.0, -1.0], [-1.0, 1.0, -1.0], [0.0, -1.0, -1.0]]))         # behind the camera
    verts = np.concatenate(tris).astype(np.float32)
    faces = np.arange(verts.shape[0]).reshape(-1, 3)
    dup = faces[g.choice(120, 60, replace=False)]
    faces = np.concatenate([faces, dup])
    faces = faces[g.permutation(faces.shape[0])]
    labels = g.integers(0, 24, faces.shape[0])
    tpose0 = g.standard_normal((verts.shape[0], 3)).astype(np.float32)
    proj = np.stack([verts, verts[:, [1, 0, 2]]])                                          # B = 2
    return proj, faces, labels, tpose0


def _check_bit_exact(proj, faces, labels, tpose0, H, W):
    pre = _pre()
    out = pre.rasterize_projected(torch.from_numpy(proj).cuda(), torch.from_numpy(faces).cuda(), torch.as_tensor(labels).cuda(),
                                  torch.from_numpy(tpose0).cuda(), H, W, debug=True)
    torch.cuda.synchronize()
    p2f, zbuf, bary = rp.rasterize(proj, faces, H, W)
    seg, sem = rp.resolve(p2f, bary, faces, labels, tpose0)
    assert (p2f >= 0).mean() > 0.05
    assert np.array_equal(out["pix_to_face"].cpu().numpy(), p2f)
    assert np.array_equal(out["zbuf"].cpu().numpy().view(np.int32), zbuf.view(np.int32))
    assert np.array_equal(out["bary"].cpu().numpy().view(np.int32), bary.view(np.int32))
    assert torch.equal(out["rasterized_segments"].cpu(), seg)
    assert torch.equal(out["rasterized_semantics"].cpu(), sem)
    return out


@pytest.mark.parametrize("H,W,B", [(512, 512, 4), (256, 128, 8)])
def test_kernels_bit_exact_on_bodies(H, W, B):
    _, faces, _, proj, labels, tpose0 = _body_case(B, H, W, seed=2)
    _check_bit_exact(proj, faces, labels, tpose0, H, W)


def test_kernels_bit_exact_on_triangle_soup():
    proj, faces, labels, tpose0 = _soup()
    p2f, _, _ = rp.rasterize(proj, faces, 64, 64)
    first = {}
    for i, f in enumerate(map(tuple, faces)):
        first.setdefault(f, i)
    won = p2f[0][p2f[0] >= 0]
    tied = [i for i in won if sum(tuple(faces[i]) == tuple(f) for f in faces[:i + 1]) == 1 and
            sum(tuple(faces[i]) == tuple(f) for f in faces) == 2]
    assert len(tied) > 0 and all(first[tuple(faces[i])] == i for i in won)     # copies exist and the lower index wins
    _check_bit_exact(proj, faces, labels, tpose0, 64, 64)


def test_projection_matches_oracle():
    cond, _, ang, proj, _, _ = _body_case(4, 256, 128, seed=3)
    R, T, focal = rp.camera(cond, ang[0], ang[1], ang[2])
    got = _pre().project(cond["vertices"].cuda(), R.cuda(), T.cuda(), focal).cpu().numpy()
    scale = np.abs(proj).max(axis=(0, 1))
    assert np.all(np.abs(got - proj) <= 1e-6 * scale)


def _device_cond(cond):
    return {k: v.cuda() for k, v in cond.items()}


def test_preprocessor_against_oracle_and_repeatable():
    pre = _pre()
    H, W, B = 256, 128, 8
    cond, faces, ang = mg.conditions(B, 4)
    labels = _labels()
    ref = rp.preprocess(cond, faces.numpy(), labels, H, W, ang[0], ang[1], ang[2])
    p = pre.Preprocessor(gen_height=H, gen_width=W).cuda()
    p.init_smpl(faces, labels)
    runs = [p.forward_with_rotation(_device_cond(cond), ang[0], ang[1], ang[2]) for _ in range(2)]
    torch.cuda.synchronize()
    for k in ("rasterized_segments", "rasterized_semantics", "cam2world_matrices"):
        assert torch.equal(runs[0][k], runs[1][k]), k
    seg = runs[0]["rasterized_segments"].cpu()
    # the device's z-buffer for the same camera (the steps of forward_with_rotation, with the debug outputs)
    smpl = importlib.import_module("3dhumangan_b200.smpl")
    dc = _device_cond(cond)
    R = torch.inverse(smpl.body_rotation(dc, ang[0], ang[1], ang[2]))
    T = dc["T"][:, :3, -1].clone()
    T[:, -1] = pre.FOCAL_RASTER / dc["scales"] * 0.5
    R_ref, T_ref, _ = rp.camera(cond, ang[0], ang[1], ang[2])
    assert float((R.cpu() - R_ref).abs().max()) < 1e-6 and float(((T.cpu() - T_ref).abs() / T_ref.abs().clamp_min(1)).max()) < 1e-6
    dbg = pre.rasterize_projected(pre.project(dc["vertices"], R, T, -pre.FOCAL_RASTER), faces.cuda(), labels.cuda(), dc["tpose_vertices"][0],
                                  H, W, debug=True)
    assert torch.equal(dbg["rasterized_segments"].cpu(), seg)
    diff = seg != ref["rasterized_segments"]
    minb = torch.from_numpy(ref["bary"]).min(-1).values
    zr, zd = torch.from_numpy(ref["zbuf"]), dbg["zbuf"].cpu()
    # The camera is ~85 units away (field of view 1 degree), where one fp32 ulp of depth is ~7.6e-6: faces of the posed surface
    # whose depths differ by an ulp or two swap when the device's torch.inverse rounds the camera differently from the CPU's.
    # So a label may differ where the oracle's pixel is on a face edge, or where both depths agree to 1e-6 (a depth tie).
    tie = (zr > 0) & (zd > 0) & ((zr - zd).abs() <= 1e-6 * zr)
    assert not bool((diff & (minb >= 1e-5) & ~tie).any())
    assert float(diff.float().mean()) <= 1e-4, float(diff.float().mean())
    c2w, _ = sp.cam2world_fix_body(cond["full_pose"], cond["R"], cond["T"], ang[0], ang[1], ang[2])
    assert float((runs[0]["cam2world_matrices"].cpu() - c2w).abs().max()) < 5e-5 * float(c2w.abs().max())
    same = torch.from_numpy(ref["pix_to_face"]).eq(dbg["pix_to_face"].cpu()) & (seg > 1)
    sem = runs[0]["rasterized_semantics"].cpu()
    # on the same face the argmax vertex can only flip where two barycentrics are (nearly) equal
    off = (sem.permute(0, 2, 3, 1)[same] != ref["rasterized_semantics"].permute(0, 2, 3, 1)[same]).any(-1)
    assert float(off.float().mean()) <= 1e-3, float(off.float().mean())


def _vertex_splat(c2w, verts, focal, H, W):
    """The mesh vertices through the generator's ray camera (oracle/port.py initial_rays: x in [-W/H, W/H] over the columns, y in
    [-1, 1] over the rows, direction (x, y, focal) in camera space), splatted and dilated by one pixel."""
    w2c = torch.inverse(c2w.double())
    p = torch.einsum("bij,bvj->bvi", w2c, F.pad(verts.double(), (0, 1), value=1.0))[..., :3]
    u = focal[:, None].double() * p[..., 0] / p[..., 2]
    v = focal[:, None].double() * p[..., 1] / p[..., 2]
    col = ((u + W / H) / (2 * W / H) * (W - 1)).round().long()
    row = ((v + 1) / 2 * (H - 1)).round().long()
    m = torch.zeros(verts.shape[0], H, W)
    ok = (col >= 0) & (col < W) & (row >= 0) & (row < H)
    for b in range(verts.shape[0]):
        m[b, row[b][ok[b]], col[b][ok[b]]] = 1
    return F.max_pool2d(m[:, None], 3, 1, 1)[:, 0] > 0


def test_silhouette_aligns_with_the_generator_camera():
    """IoU of the rasterised silhouette with the generator camera's projection of the vertices: 0.894 on the CPU oracle for this
    case; the map mirrored left-right or up-down scores about 0.56 there."""
    pre = _pre()
    H, W, B = 256, 128, 4
    cond, faces, ang = mg.conditions(B, 7)
    p = pre.Preprocessor(gen_height=H, gen_width=W).cuda()
    p.init_smpl(faces, _labels())
    out = p.forward_with_rotation(_device_cond(cond), ang[0], ang[1], ang[2])
    sil = out["rasterized_segments"].cpu() > 1
    splat = _vertex_splat(out["cam2world_matrices"].cpu(), cond["vertices"], cond["intrinsics"][:, 0, 0], H, W)
    iou = lambda a: float((a & splat).sum()) / float((a | splat).sum())
    assert iou(sil) >= 0.88, iou(sil)
    assert iou(sil.flip(-1)) < iou(sil) - 0.2 and iou(sil.flip(-2)) < iou(sil) - 0.2, (iou(sil.flip(-1)), iou(sil.flip(-2)))


def _tiny_setup(pkg):
    gen = importlib.import_module("3dhumangan_b200.modules.generator")
    disc = importlib.import_module("3dhumangan_b200.modules.discriminator")
    smpl = importlib.import_module("3dhumangan_b200.smpl")
    cfg = pkg.configs.baseline_config("tiny")
    torch.manual_seed(0)
    G = gen.Map3DGenerator(**cfg).cuda()
    G.set_device(torch.device("cuda:0"))
    D = disc.UNetDiscriminator(**cfg).cuda()
    model, faces = smpl.SMPLModel.synthetic_surface("cuda", seed=1)
    B = 2
    g = torch.Generator().manual_seed(9)
    out = smpl.lbs(torch.randn(B, 10, generator=g) * 0.5, torch.randn(B, 24, 3, generator=g) * 0.15, model)
    cond = smpl.conditions_fix_body(torch.tensor([[1.3, 1.0, 0.02, -0.03]] * B), out, model)
    cond["cam2world_matrices"] = smpl.cam2world_fix_body(cond, torch.zeros(B), torch.zeros(B), torch.zeros(B))
    batch = {"images": torch.rand(B, 3, cfg["gen_height"], cfg["gen_width"], device="cuda") * 2 - 1,
             "labels": torch.randint(2, 26, (B, cfg["gen_height"], cfg["gen_width"]), device="cuda"), "cond": cond}
    return cfg, G, D, faces, batch


@pytest.mark.parametrize("rotate", [True, False])
def test_trainer_uses_rasterised_targets_on_the_reference_schedule(pkg, rotate):
    pre = _pre()
    ts = importlib.import_module("3dhumangan_b200.train_step")
    cfg, G, D, faces, batch = _tiny_setup(pkg)
    cfg["phases"] = [dict(p, rotate=rotate, do_r1=False) for p in cfg["phases"]]
    p = pre.Preprocessor(**cfg).cuda()
    p.init_smpl(faces, _labels())
    t = ts.Trainer(G, D, cfg, amp=False, preprocessor=p)
    seen = []
    orig = t._seg_loss
    t._seg_loss = lambda s, gt: (seen.append(gt.detach().clone()), orig(s, gt))[1]
    real_pp = p.forward
    maps = []
    p.forward = lambda data, r=False, **kw: (lambda d: (maps.append(d["rasterized_segments"].clone()), d)[1])(real_pp(data, r, **kw))
    # the reference draws random.random() only where the phase does not rotate: D target, then G target
    random.seed(11)
    draws = [] if rotate else [random.random(), random.random()]
    random.seed(11)
    torch.manual_seed(12)
    d, gl = t.iteration(batch)
    torch.cuda.synchronize()
    assert bool(torch.isfinite(d)) and bool(torch.isfinite(gl))
    assert len(maps) == 2 and len(seen) == 3           # D: real + gen targets, G: one split
    assert all(bool((m > 1).any()) and bool((m == 1).any()) for m in maps)
    use = [True, True] if rotate else [x < 0.5 for x in draws]
    assert torch.equal(seen[0], maps[0] if use[0] else batch["labels"])
    assert torch.equal(seen[1], torch.zeros_like(batch["labels"]))
    assert torch.equal(seen[2], maps[1] if use[1] else batch["labels"])
    assert "rasterized_segments" not in batch["cond"]          # the caller's conditions are not modified


def _semantic_frame(sem):
    """apps/sample_from_generator.py:53-56 and :64-65: clamp, background (all zero) -> 1, then to uint8 HWC."""
    smpl = torch.clamp(sem, -1, 1)
    bg = torch.all(smpl == 0, dim=1, keepdim=True)
    smpl[bg.repeat(1, 3, 1, 1)] = 1
    return torch.clamp((smpl * 0.5 + 0.5) * 255, 0, 255).to(torch.uint8).permute(0, 2, 3, 1).cpu().numpy()


def test_sample_replay_with_stitched_semantics():
    """`generate_frames` (apps/sample_from_generator.py:24-67) drives `forward_with_rotation` one sample per frame with [1,1]
    angle tensors on the device (a turn-table of +-pi/6), and --stitch (:136-138) stacks each frame on its semantics image.
    Replayed here with the device preprocessor and with the oracle: the stitched semantic frames agree outside label-edge
    pixels."""
    pre = _pre()
    H, W, n = 256, 128, 5
    cond, faces, _ = mg.conditions(1, 6)
    labels = _labels()
    p = pre.Preprocessor(gen_height=H, gen_width=W).cuda()
    p.init_smpl(faces, labels)
    conds = {k: v.repeat_interleave(n, dim=0).cuda() for k, v in cond.items()}
    angles_h = torch.linspace(-np.pi / 6, np.pi / 6, n, device="cuda").unsqueeze(-1)
    angles_v = torch.linspace(0, 0, n, device="cuda").unsqueeze(-1)
    angles_r = torch.zeros_like(angles_h)
    frames = []
    for i in range(n):
        sub = {k: v[i:i + 1] for k, v in conds.items()}
        sub = p.forward_with_rotation(sub, angles_h[i:i + 1], angles_v[i:i + 1], angles_r[i:i + 1])
        got = _semantic_frame(sub["rasterized_semantics"])[0]
        ref = rp.preprocess(cond, faces.numpy(), labels, H, W, angles_h[i].cpu(), angles_v[i].cpu(), angles_r[i].cpu())
        want = _semantic_frame(ref["rasterized_semantics"])[0]
        assert np.any(got != 255)
        assert np.mean(np.any(got != want, -1)) <= 1e-4
        stitched = np.concatenate([np.zeros((H, W, 3), np.uint8), got], axis=0)
        assert stitched.shape == (2 * H, W, 3)
        frames.append(got)
    assert not np.array_equal(frames[0], frames[-1])
