"""ctypes binding of the C ABI declared in include/hg3d.h.

The product path has NO fallback: if `lib3dhg_sm90a.so` is missing, fails to load, or an entry
point returns non-zero, a RuntimeError is raised (mirroring TORCH_CHECK -> RuntimeError in the
reference's own native ops, lib/components/ops/bias_act.cpp:34-51).  All pointers are raw device
pointers taken from torch tensors; the library never allocates device memory and never
synchronises the device; the CUDA stream is passed explicitly (torch's current stream).
"""
from __future__ import annotations

import ctypes
import os
from ctypes import c_char_p, c_double, c_float, c_int, c_long, c_size_t, c_void_p

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib3dhg_sm90a.so")
_lib = None

# name -> (restype, argtypes).  Keep in sync with include/hg3d.h (tests check every symbol).
SIGNATURES = {
    "hg_last_error": (c_char_p, []),
    "hg_abi_version": (c_int, []),
    "hg_check_device": (c_int, []),
    "hg_packed_weight_bytes": (c_size_t, [c_int, c_int, c_int]),
    "hg_pack_weight": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_float, c_int, c_void_p, c_size_t, c_void_p]),
    "hg_vertex_ik": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p]),
    "hg_knn_padded": (c_int, [c_int]),
    "hg_knn_prep": (c_int, [c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "hg_geo_features": (c_int, [c_void_p] * 14 + [c_int] * 6 + [c_float, c_int] + [c_void_p] * 6),
    "hg_sample_fine": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_float, c_int] + [c_void_p] * 4 + [c_int] * 4
                       + [c_void_p] * 3),
    "hg_merge_samples": (c_int, [c_void_p] * 4 + [c_int] * 3 + [c_void_p] * 4),
    "hg_iso_workspace_bytes": (c_size_t, [c_int, c_int, c_int]),
    "hg_iso_count": (c_int, [c_void_p, c_int, c_int, c_int, c_float, c_void_p, c_size_t, c_void_p, c_void_p]),
    "hg_iso_emit": (c_int, [c_void_p, c_int, c_int, c_int] + [c_float] * 5 + [c_void_p, c_size_t, ctypes.c_longlong]
                    + [c_void_p] * 4),
    "hg_spade_conv": (c_int, [c_void_p, c_long, c_void_p, c_void_p, c_void_p, c_long] + [c_void_p] * 12 + [c_int] * 7 + [c_void_p]),
    "hg_bn_finalize": (c_int, [c_void_p, c_double, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_float, c_float,
                               c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "hg_synth_input": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_void_p]),
    "hg_render_weight_blob_bytes": (c_size_t, []),
    "hg_render_mlp": (c_int, [c_void_p] * 12 + [c_int] * 4 + [c_float] + [c_int] * 4 + [c_void_p]),
    "hg_spade_bwd_dgrad": (c_int, [c_void_p, c_void_p, c_long, c_void_p, c_void_p, c_void_p, c_void_p] + [c_int] * 5 + [c_void_p]),
    "hg_spade_bwd_wgrad_workspace_bytes": (c_size_t, []),
    "hg_spade_bwd_wgrad": (c_int, [c_void_p, c_void_p, c_long, c_void_p, c_void_p, c_void_p, c_void_p] + [c_int] * 5 + [c_void_p]),
    "hg_spade_bwd_combine": (c_int, [c_void_p, c_void_p, c_long] + [c_void_p] * 7 + [c_int] * 4 + [c_void_p]),
    "hg_conv1x1_blocked": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p] + [c_int] * 4 + [c_void_p]),
    "hg_conv1x1_blocked_bwd": (c_int, [c_void_p] * 7 + [c_int, c_float, c_int, c_int, c_void_p, c_void_p, c_void_p, c_int]
                               + [c_int] * 4 + [c_void_p]),
    "hg_act_conv1x1_blocked": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p] + [c_int] * 4 + [c_void_p]),
    "hg_act_wgrad_blocked": (c_int, [c_void_p, c_void_p, c_void_p, c_long, c_int, c_void_p, c_int, c_void_p, c_void_p, c_void_p]
                             + [c_int] * 5 + [c_void_p]),
    "hg_render_heads": (c_int, [c_void_p] * 8 + [c_int, c_int, c_void_p]),
    "hg_render_heads_bwd": (c_int, [c_void_p] * 6 + [c_int, c_int, c_void_p]),
    "hg_render_composite": (c_int, [c_void_p] * 7 + [c_int, c_int, c_int, c_float, c_int, c_int, c_int, c_void_p]),
    "hg_blocked_conv_wide": (c_int, [c_void_p] * 4 + [c_int, c_float] + [c_void_p] * 9 + [c_int] * 4 + [c_void_p]),
    "hg_render_composite_bwd": (c_int, [c_void_p] * 9 + [c_int, c_int, c_int, c_float, c_int, c_int, c_int, c_void_p]),
    "hg_wgrad_blocked": (c_int, [c_void_p, c_void_p, c_long, c_int, c_void_p, c_void_p, c_void_p, c_void_p] + [c_int] * 5 + [c_void_p]),
    "hg_spade_a1": (c_int, [c_void_p, c_long, c_void_p, c_void_p] + [c_int] * 5 + [c_void_p]),
    "hg_spade_pixel_pre": (c_int, [c_void_p, c_long, c_void_p, c_void_p, c_void_p] + [c_int] * 4 + [c_void_p]),
    "hg_spade_pixel_mod_bwd": (c_int, [c_void_p, c_void_p, c_long, c_void_p, c_void_p, c_void_p, c_void_p] + [c_int] * 4 + [c_void_p]),
    "hg_bilinear_adjoint": (c_int, [c_void_p, c_void_p, c_long] + [c_int] * 5 + [c_void_p]),
    "hg_conv2d_wgrad_workspace_bytes": (c_size_t, []),
    "hg_conv2d_wgrad_taps": (c_int, [c_void_p] * 5 + [c_int] * 10 + [c_void_p, c_void_p, c_int, c_void_p]),
    "hg_conv2d_wgrad_layer_workspace_bytes": (c_size_t, [c_int] * 6),
    "hg_conv2d_wgrad_layer": (c_int, [c_void_p] * 5 + [c_size_t] + [c_int] * 7 + [c_void_p]),
    "hg_synth_input_bwd": (c_int, [c_void_p] * 5 + [c_int] * 4 + [c_void_p, c_void_p, c_void_p]),
    "hg_bias_act": (c_int, [c_void_p, c_void_p, c_void_p, c_long, c_int, c_int, c_int, c_float, c_float, c_float, c_void_p]),
    "hg_bias_act_grad": (c_int, [c_void_p] * 6 + [c_long, c_int, c_int, c_int, c_int, c_float, c_float, c_float, c_void_p]),
    "hg_resample2x": (c_int, [c_void_p, c_void_p, c_long, c_int, c_int, c_int, c_float, c_void_p]),
    "hg_upfirdn2d": (c_int, [c_void_p, c_void_p, c_void_p] + [c_int] * 14 + [c_float, c_void_p]),
    "hg_upfirdn2d_sep2": (c_int, [c_void_p, c_void_p, c_void_p, c_long] + [c_int] * 9 + [c_float, c_void_p]),
    "hg_conv2d": (c_int, [c_void_p, c_int, c_void_p, c_int] + [c_int] * 6 + [c_void_p, c_int, c_int, c_void_p, c_void_p, c_int,
                              c_void_p, c_int, c_void_p]),
    "hg_pool_add": (c_int, [c_void_p, c_int, c_void_p, c_int, c_void_p, c_long, c_int, c_int, c_void_p]),
    "hg_dense": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]),
    "hg_linear": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_int, c_int, c_void_p, c_void_p, c_int, c_int, c_void_p]),
    "hg_conv3x3_wgrad_halo_workspace_bytes": (ctypes.c_size_t, []),
    "hg_conv3x3_wgrad_halo": (c_int, [c_void_p] * 5 + [c_int] * 10 + [c_void_p, c_void_p, c_int, c_void_p]),
    "hg_label_histogram": (c_int, [c_void_p, c_long, c_int, c_void_p, c_void_p]),
    "hg_seg_ce_coef": (c_int, [c_void_p, c_void_p, c_int, c_double, c_void_p, c_void_p]),
    "hg_seg_ce": (c_int, [c_void_p] * 6 + [c_int, c_int, c_long, c_void_p]),
    "hg_image_loss": (c_int, [c_void_p] * 6 + [c_int, c_long, c_int, c_float, c_void_p]),
    "hg_latent_pool_gather": (c_int, [c_void_p, c_long, c_int, c_void_p, c_int, c_void_p, c_void_p]),
    "hg_latent_pool_grad": (c_int, [c_void_p, c_void_p, c_int, c_int, c_long, c_void_p, c_void_p]),
    "hg_latent_loss": (c_int, [c_void_p, c_void_p, c_int, c_int, c_float, c_void_p, c_void_p, c_void_p, c_void_p]),
    "hg_vgg_input": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p]),
    "hg_vgg_input_adjoint": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]),
    "hg_maxpool2x2": (c_int, [c_void_p, c_void_p, c_long, c_int, c_int, c_void_p]),
    "hg_vgg_level_bwd": (c_int, [c_void_p] * 4 + [c_float, c_void_p, c_long, c_int, c_int, c_void_p]),
    "hg_smooth_l1": (c_int, [c_void_p, c_void_p, c_long, c_void_p, c_void_p, c_void_p]),
    "hg_mt_entry_bytes": (c_int, []),
    "hg_mt_chunk_bytes": (c_int, []),
    "hg_mt_chunk_elems": (c_int, []),
    "hg_mt_grad_norm": (c_int, [c_void_p, c_void_p, c_int, c_float, c_void_p, c_void_p, c_void_p]),
    "hg_mt_adam": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_int, c_float, c_int, c_void_p]),
    "hg_smpl_shape_blocks": (c_int, [c_int]),
    "hg_smpl_shape": (c_int, [c_void_p] * 6 + [c_int] * 4 + [c_void_p]),
    "hg_smpl_pose": (c_int, [c_void_p, c_int, c_void_p, c_int] + [c_void_p] * 6 + [c_int, c_int, c_void_p]),
    "hg_smpl_skin": (c_int, [c_void_p, c_long, c_void_p, c_void_p, c_int, c_void_p, c_long, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]),
    "hg_raster_project": (c_int, [c_void_p, c_void_p, c_void_p, c_float, c_void_p, c_int, c_int, c_void_p]),
    "hg_raster_faces": (c_int, [c_void_p, c_void_p] + [c_int] * 5 + [c_void_p, c_void_p]),
    "hg_raster_resolve": (c_int, [c_void_p] * 5 + [c_int] * 5 + [c_void_p] * 6),
    "hg_spectral_entry_bytes": (c_int, []),
    "hg_spectral_norm": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_int, c_float, c_void_p]),
}


def lib():
    """Load the shared library once; raise loudly when it is absent (no CPU / eager fallback)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} not found: build it with `python 3dhumangan_b200/build.py` "
                "(this package has no CPU or eager-PyTorch fallback)")
        handle = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(handle, name)
            fn.restype = res
            fn.argtypes = args
        _lib = handle
    return _lib


def check(rc: int, what: str):
    if rc != 0:
        msg = lib().hg_last_error().decode("utf-8", "replace")
        raise RuntimeError(f"{what} failed (code {rc}): {msg}")


LAUNCHES = 0        # kernels launched through this binding (bench.py reports it as gpu_launches)
TIMING = None       # when a list: (name, start_event, end_event) per launch, recorded on the current stream
TIMING_TAGS = False # tools: record "name[tag]" (layer shapes) instead of the bare entry-point name


def call(name, *args, tag=None):
    """Invoke one launching entry point: count it, optionally bracket it with CUDA events, raise on error."""
    global LAUNCHES
    fn = getattr(lib(), name)
    if TIMING is not None:
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        rc = fn(*args)
        e.record()
        TIMING.append((f"{name}[{tag}]" if TIMING_TAGS and tag else name, s, e))
    else:
        rc = fn(*args)
    LAUNCHES += 1
    check(rc, name)


def ptr(t):
    """Device pointer of a tensor (or NULL).  Tensors must be CUDA + contiguous."""
    if t is None:
        return None
    if not t.is_cuda:
        raise RuntimeError("hg3d: expected a CUDA tensor (there is no CPU path)")
    if not t.is_contiguous():
        raise RuntimeError("hg3d: expected a contiguous tensor")
    return c_void_p(t.data_ptr())


def stream():
    return c_void_p(torch.cuda.current_stream().cuda_stream)


_DEVICE_OK = set()


def require_device(t=None):
    if not torch.cuda.is_available():
        raise RuntimeError("hg3d: no CUDA device visible; the sm_90a kernels cannot run (no fallback)")
    dev = torch.cuda.current_device()
    if dev not in _DEVICE_OK:          # cudaGetDeviceProperties is slow: check each device once
        check(lib().hg_check_device(), "hg_check_device")
        _DEVICE_OK.add(dev)


# ----------------------------------------------------------------------------------------------
# thin typed wrappers (shape checks live in C; these only marshal)
# ----------------------------------------------------------------------------------------------
def packed_weight_bytes(N, K, Nb):
    return int(lib().hg_packed_weight_bytes(N, K, Nb))


def pack_weight(W, Nb=None, scale=1.0, scale_dev=None, out=None):
    """W [N,K] fp32 (row stride may exceed K) -> packed bf16 hi/lo operand image (uint8 tensor)."""
    assert W.dim() == 2 and W.dtype == torch.float32 and W.stride(1) == 1
    N, K = W.shape
    if Nb is None:
        Nb = min(256, (N + 15) // 16 * 16)
    nbytes = packed_weight_bytes(N, K, Nb)
    if out is None:
        out = torch.empty(nbytes, dtype=torch.uint8, device=W.device)
    with torch.cuda.device_of(W):
        call("hg_pack_weight", c_void_p(W.data_ptr()), N, K, W.stride(0), ptr(scale_dev), float(scale), Nb,
                                   ptr(out), out.numel(), stream())
    return out, Nb


def linear(X, Wimg, Nb, N, bias=None, passes=3, out=None):
    """Y = X @ W^T + bias with the packed weight image; X [M,K] fp32 row-major."""
    assert X.dim() == 2 and X.dtype == torch.float32 and X.stride(1) == 1
    M, K = X.shape
    if out is None:
        out = torch.empty(M, N, dtype=torch.float32, device=X.device)
    with torch.cuda.device_of(X):
        call("hg_linear", c_void_p(X.data_ptr()), X.stride(0), M, K, ptr(Wimg), Nb, N, ptr(bias),
                              ptr(out), out.stride(0), passes, stream())
    return out


_SN_TABLES = {}


def spectral_norm(ws, us, vs, training, eps=1e-12):
    """One launch for a list of weights: power iteration (training: u / v buffers updated in place) and 1/sigma.
    ws: tensors whose first dim is N (viewed as [N, K]), us [N], vs [K].  Returns inv_sigma [n] fp32."""
    import numpy as np
    dev = ws[0].device
    key = tuple((w.data_ptr(), u.data_ptr(), v.data_ptr(), w.shape[0], w.numel() // w.shape[0]) for w, u, v in zip(ws, us, vs))
    ent = _SN_TABLES.get(key)
    if ent is None:
        assert int(lib().hg_spectral_entry_bytes()) == 32
        for w, u, v in zip(ws, us, vs):
            assert w.is_contiguous() and u.is_contiguous() and v.is_contiguous() and w.dtype == u.dtype == v.dtype == torch.float32
        tab = np.zeros((len(ws), 4), dtype=np.int64)
        for i, (w_, u_, v_, n, k) in enumerate(key):
            tab[i] = (w_, u_, v_, n | (k << 32))
        if len(_SN_TABLES) > 64:
            _SN_TABLES.clear()
        ent = _SN_TABLES[key] = (torch.from_numpy(tab).to(dev), max(k_[3] for k_ in key), max(k_[4] for k_ in key))
    table, max_n, max_k = ent
    inv = torch.empty(len(ws), dtype=torch.float32, device=dev)
    with torch.cuda.device_of(inv):
        call("hg_spectral_norm", ptr(table), len(ws), max_n, max_k, ptr(inv), int(bool(training)), float(eps), stream())
    return inv


def vertex_ik(fk, lbs):
    """fk [B,24,4,4], lbs [B,V,24] -> [B,V,16] blended inverse transforms (smpl.py:217-218)."""
    B, V = lbs.shape[0], lbs.shape[1]
    fk = fk.float().contiguous()
    lbs = lbs.float().contiguous()
    out = torch.empty(B, V, 16, dtype=torch.float32, device=fk.device)
    with torch.cuda.device_of(fk):
        call("hg_vertex_ik", ptr(fk), ptr(lbs), B, V, ptr(out), stream())
    return out


def geo_features(cond_vertices, tpose, skeletons, vik, *, input_scaler, legacy_mode=False, points_in=None,
                 xs=None, ys=None, zs=None, focals=None, scales=None, cam2world=None, jitter=None,
                 want_points=False, want_nearest=False, brute_force=False):
    """Ray sampling (or given points) + K=1 nearest vertex + 31-d features -> point records [B,N,36].

    Returns dict(rec, z_vals, points, nearest, nearest_d2) (optional outputs None unless requested)."""
    dev = cond_vertices.device
    B, V = cond_vertices.shape[0], cond_vertices.shape[1]
    f = lambda t: None if t is None else t.float().contiguous()
    if points_in is not None:
        points_in = f(points_in)
        N, Rw, Rh, S = points_in.shape[1], 0, 0, 0
    else:
        Rw, Rh, S = xs.numel(), ys.numel(), zs.numel()
        N = Rw * Rh * S
    rec = torch.empty(B, N, 36, dtype=torch.float32, device=dev)
    z_vals = torch.empty(B, N, dtype=torch.float32, device=dev) if points_in is None else None
    pts = torch.empty(B, N, 3, dtype=torch.float32, device=dev) if want_points else None
    near = torch.empty(B, N, dtype=torch.int32, device=dev) if want_nearest else None
    d2 = torch.empty(B, N, dtype=torch.float32, device=dev) if want_nearest else None
    verts = f(cond_vertices)
    ksort = kbox = None
    if not brute_force and V <= 8192:
        Vp = int(lib().hg_knn_padded(V))
        ksort = torch.empty(B, Vp, 4, dtype=torch.float32, device=dev)
        kbox = torch.empty(B, Vp // 32, 2, 4, dtype=torch.float32, device=dev)
        with torch.cuda.device_of(rec):
            call("hg_knn_prep", ptr(verts), B, V, ptr(ksort), ptr(kbox), stream())
    keep = [f(t) for t in (xs, ys, zs, focals, scales, cam2world, jitter, points_in, skeletons, verts, tpose, vik)]
    keep += [ksort, kbox]
    with torch.cuda.device_of(rec):
        call("hg_geo_features", *[ptr(t) for t in keep], B, Rw, Rh, S, V, N, float(input_scaler),
                                    int(bool(legacy_mode)), ptr(rec), ptr(z_vals), ptr(pts), ptr(near), ptr(d2),
                                    stream())
    return {"rec": rec, "z_vals": z_vals, "points": pts, "nearest": near, "nearest_d2": d2}


def sample_fine(sigma, sigma_stride, z_vals, noise, u_pdf, *, noise_std, clamp_mode, xs, ys, focals, cam2world, B, Rw, Rh, S):
    """Coarse weights + inverse-cdf sampling of hierarchical_sample (csrc/sample.cu) -> fine z [B,R*S], points [B,R*S,3].
    `sigma` is read at p * sigma_stride for point p (the sigma column of a per-point output can be passed as a view)."""
    dev = z_vals.device
    if clamp_mode not in ("relu", "softplus"):
        raise RuntimeError("Need to choose clamp mode")          # volume_rendering.py:31
    f = lambda t: None if t is None else t.float().contiguous()
    keep = [f(t) for t in (z_vals, noise, u_pdf, xs, ys, focals, cam2world)]
    fine_z = torch.empty(B, Rw * Rh * S, dtype=torch.float32, device=dev)
    pts = torch.empty(B, Rw * Rh * S, 3, dtype=torch.float32, device=dev)
    if not sigma.is_cuda:
        raise RuntimeError("hg3d: expected a CUDA tensor (there is no CPU path)")
    with torch.cuda.device_of(fine_z):
        call("hg_sample_fine", c_void_p(sigma.data_ptr()), int(sigma_stride), ptr(keep[0]), ptr(keep[1]), ptr(keep[2]),
             float(noise_std), int(clamp_mode == "softplus"), *[ptr(t) for t in keep[3:]], B, Rw, Rh, S, ptr(fine_z), ptr(pts),
             stream())
    return fine_z, pts


def merge_samples(fine_rec, fine_z, coarse_rec, coarse_z, *, B, R, S, want_perm=False):
    """Depth-sorted merge of the fine and coarse samples of every ray (csrc/sample.cu) -> rec [B,R*2S,36], z [B,R*2S],
    perm [B,R*2S] int32 (index into cat([fine, coarse]) per ray) or None."""
    dev = fine_rec.device
    rec = torch.empty(B, R * 2 * S, 36, dtype=torch.float32, device=dev)
    z = torch.empty(B, R * 2 * S, dtype=torch.float32, device=dev)
    perm = torch.empty(B, R * 2 * S, dtype=torch.int32, device=dev) if want_perm else None
    with torch.cuda.device_of(rec):
        call("hg_merge_samples", ptr(fine_rec), ptr(fine_z), ptr(coarse_rec), ptr(coarse_z), B, R, S, ptr(rec), ptr(z), ptr(perm),
             stream())
    return rec, z, perm


def spade_conv(x, x_bstride, wimg, bias, out, *, B, Hg, Wg, mod=None, scsh=None, p_lr=None, p_stride=0, p_bias=None,
               wgb=None, bgb=None, skip=None, stats=None, rgb_w=None, rgb_b=None, rgb_in=None, rgb_out=None,
               Rh=0, Rw=0, passes=3):
    """One SPADE half-block (see csrc/synth.cu).  All tensors fp32 CUDA; `stats` is a float64 view [>=512]."""
    tag = None
    if TIMING_TAGS:
        flags = "".join(f" {n}" for n, t in (("skip", skip), ("rgb", rgb_w), ("stats", stats)) if t is not None)
        flags += " xshared" if x_bstride == 0 else ""
        tag = f"{'pixel' if p_lr is not None else 'const'}{flags} {Hg}x{Wg} B{B}"
    with torch.cuda.device_of(out):
        call("hg_spade_conv", ptr(x), int(x_bstride), ptr(mod), ptr(scsh), ptr(p_lr), int(p_stride), ptr(p_bias),
                                  ptr(wgb), ptr(bgb), ptr(wimg), ptr(bias), ptr(skip), ptr(out), ptr(stats),
                                  ptr(rgb_w), ptr(rgb_b), ptr(rgb_in), ptr(rgb_out), B, 256, Hg, Wg, Rh, Rw, passes,
                                  stream(), tag=tag)
    return out


def spade_bwd_dgrad(dout, x, x_bstride, mod, wimg_t, dpre, sums, *, B, Hg, Wg, passes=3):
    """dpre = (W^T dout) * lrelu'(x*g1+g0); sums [B,2,C] float64 += (sum dpre, sum dpre*x)  (csrc/synth.cu)."""
    with torch.cuda.device_of(dout):
        call("hg_spade_bwd_dgrad", ptr(dout), ptr(x), int(x_bstride), ptr(mod), ptr(wimg_t), ptr(dpre), ptr(sums), B, 256,
             Hg, Wg, passes, stream())
    return dpre


_WGRAD_WS = {}


def spade_bwd_wgrad(dout, x, x_bstride, mod, *, B, Hg, Wg, passes=3, want_bias=True, Cx=256):
    """dW [C,Cx] = sum dout (x) lrelu(x*g1+g0), dbias [C] = sum dout  (csrc/synth_bwd.cu); mod None: y = lrelu(x)."""
    dev = dout.device
    ws = _WGRAD_WS.get(dev)
    if ws is None:
        ws = _WGRAD_WS[dev] = torch.empty(int(lib().hg_spade_bwd_wgrad_workspace_bytes()) // 4, dtype=torch.float32, device=dev)
    dw = torch.empty(256, Cx, dtype=torch.float32, device=dev)
    db = torch.empty(256, dtype=torch.float32, device=dev) if want_bias else None
    with torch.cuda.device_of(dout):
        call("hg_wgrad_blocked", ptr(dout), ptr(x), int(x_bstride), Cx, ptr(mod), ptr(dw), ptr(db), ptr(ws), B, 256, Hg, Wg,
             passes, stream())
    return dw, db


def conv1x1_blocked(x, Cin, wimg, bias, out, *, B, Hg, Wg, passes=3):
    with torch.cuda.device_of(x):
        call("hg_conv1x1_blocked", ptr(x), Cin, ptr(wimg), ptr(bias), ptr(out), B, Hg, Wg, passes, stream())
    return out


def conv1x1_blocked_bwd(g, aux, wimg_t, out, sums, *, B, Hg, Wg, g2=None, mod=None, Cout=256, slope=0.2, pixel_major=False,
                        passes=3, act=0, ascale=None, rk_w=None, rk_v=None):
    rk_n = 0 if rk_v is None else rk_v.shape[1]
    with torch.cuda.device_of(g):
        call("hg_conv1x1_blocked_bwd", ptr(g), ptr(g2), ptr(aux), ptr(mod), ptr(wimg_t), ptr(out), ptr(sums), Cout,
             float(slope), int(bool(pixel_major)), act, ptr(ascale), ptr(rk_w), ptr(rk_v), rk_n, B, Hg, Wg, passes, stream())
    return out


def act_conv1x1_blocked(x, mod, wimg, bias, out, *, B, Hg, Wg, x2=None, act=1, passes=3):
    """out = W [act(x*g1+g0); act(x2*g1+g0)] + bias over tile-blocked points / pixels (act 1 = sine)."""
    with torch.cuda.device_of(x):
        call("hg_act_conv1x1_blocked", ptr(x), ptr(x2), ptr(mod), act, ptr(wimg), ptr(bias), ptr(out), B, Hg, Wg, passes, stream())
    return out


def act_wgrad_blocked(dout, x, x_bstride, mod, *, B, Hg, Wg, act, pscale=None, Cx=256, passes=3):
    dev = dout.device
    ws = _WGRAD_WS.get(dev)
    if ws is None:
        ws = _WGRAD_WS[dev] = torch.empty(int(lib().hg_spade_bwd_wgrad_workspace_bytes()) // 4, dtype=torch.float32, device=dev)
    dw = torch.empty(256, Cx, dtype=torch.float32, device=dev)
    db = torch.empty(256, dtype=torch.float32, device=dev)
    with torch.cuda.device_of(dout):
        call("hg_act_wgrad_blocked", ptr(dout), ptr(pscale), ptr(x), int(x_bstride), Cx, ptr(mod), act, ptr(dw), ptr(db), ptr(ws),
             B, 256, Hg, Wg, passes, stream())
    return dw, db


def render_heads(out3, linc, mod3, w_sigma, w_rgb, heads_b, *, B, N):
    sig = torch.empty(B, N, dtype=torch.float32, device=out3.device)
    rgbp = torch.empty(B, 3, N, dtype=torch.float32, device=out3.device)
    with torch.cuda.device_of(out3):
        call("hg_render_heads", ptr(out3), ptr(linc), ptr(mod3), ptr(w_sigma), ptr(w_rgb), ptr(heads_b), ptr(sig), ptr(rgbp), B, N,
             stream())
    return sig, rgbp


def render_heads_bwd(out3, linc, mod3, dsig, drgbp, *, B, N):
    acc = torch.zeros(4 * 256 + 4, dtype=torch.float64, device=out3.device)
    with torch.cuda.device_of(out3):
        call("hg_render_heads_bwd", ptr(out3), ptr(linc), ptr(mod3), ptr(dsig), ptr(drgbp), ptr(acc), B, N, stream())
    return acc


def render_composite(sig, z, noise, rgbp, feat, *, B, R, S, noise_std, white_back, softplus, last_back=False):
    ray_out = torch.empty(B, R, 260, dtype=torch.float32, device=sig.device)
    w = torch.empty(B, R * S, dtype=torch.float32, device=sig.device)
    with torch.cuda.device_of(sig):
        call("hg_render_composite", ptr(sig), ptr(z), ptr(noise), ptr(rgbp), ptr(feat), ptr(ray_out), ptr(w), B, R, S,
             float(noise_std), int(bool(white_back)), int(bool(softplus)), int(bool(last_back)), stream())
    return ray_out, w


def render_composite_bwd(sig, z, noise, rgbp, feat, dray, *, B, R, S, noise_std, white_back, softplus, last_back=False):
    dfeat = torch.empty_like(feat)
    drgbp = torch.empty_like(rgbp)
    dsig = torch.empty_like(sig)
    with torch.cuda.device_of(sig):
        call("hg_render_composite_bwd", ptr(sig), ptr(z), ptr(noise), ptr(rgbp), ptr(feat), ptr(dray), ptr(dfeat), ptr(drgbp),
             ptr(dsig), B, R, S, float(noise_std), int(bool(white_back)), int(bool(softplus)), int(bool(last_back)), stream())
    return dfeat, drgbp, dsig


def spade_a1(p_lr, p_stride, p_bias, a1, *, B, Hg, Wg, Rh, Rw):
    with torch.cuda.device_of(a1):
        call("hg_spade_a1", ptr(p_lr), int(p_stride), ptr(p_bias), ptr(a1), B, Hg, Wg, Rh, Rw, stream())
    return a1


def spade_pixel_pre(x, x_bstride, scsh, gam, bet_pre, *, B, Hg, Wg):
    with torch.cuda.device_of(gam):
        call("hg_spade_pixel_pre", ptr(x), int(x_bstride), ptr(scsh), ptr(gam), ptr(bet_pre), B, 256, Hg, Wg, stream())
    return bet_pre


def spade_pixel_mod_bwd(dpre, x, x_bstride, scsh, gam_dgam, dxn, sums, *, B, Hg, Wg):
    with torch.cuda.device_of(dpre):
        call("hg_spade_pixel_mod_bwd", ptr(dpre), ptr(x), int(x_bstride), ptr(scsh), ptr(gam_dgam), ptr(dxn), ptr(sums), B, 256,
             Hg, Wg, stream())


def bilinear_adjoint(da1, dp, dp_stride, *, B, Hg, Wg, Rh, Rw):
    with torch.cuda.device_of(da1):
        call("hg_bilinear_adjoint", ptr(da1), ptr(dp), int(dp_stride), B, Hg, Wg, Rh, Rw, stream())


def spade_bwd_combine(dx, *, B, Hg, Wg, dpre=None, x=None, x_bstride=0, g1=None, ak=None, dskip=None, drgb=None, rgb_w=None,
                      dwrgb=None):
    """dx = dpre*g1 + a + k*x (+ dskip) (+ rgb_w^T drgb); dwrgb [3,C] float64 += drgb . x^T  (csrc/synth_bwd.cu)."""
    with torch.cuda.device_of(dx):
        call("hg_spade_bwd_combine", ptr(dpre), ptr(x), int(x_bstride), ptr(g1), ptr(ak), ptr(dskip), ptr(drgb), ptr(rgb_w),
             ptr(dx), ptr(dwrgb), B, 256, Hg, Wg, stream())
    return dx


def synth_input_bwd(dx, w, bias, ic, jc, B):
    C = w.shape[0]
    dw = torch.empty(C, 2, dtype=torch.float32, device=dx.device)
    db = torch.empty(C, dtype=torch.float32, device=dx.device)
    with torch.cuda.device_of(dx):
        call("hg_synth_input_bwd", ptr(dx), ptr(w), ptr(bias), ptr(ic), ptr(jc), B, C, ic.numel(), jc.numel(), ptr(dw), ptr(db),
             stream())
    return dw, db


def bn_finalize(stats, weight, bias, running_mean, running_var, training, *, count=0.0, count_dev=None, gb=None, B=0,
                scsh=None, mod=None, eps=1e-5, momentum=0.1):
    with torch.cuda.device_of(weight):
        call("hg_bn_finalize", ptr(stats), float(count), ptr(count_dev), ptr(weight), ptr(bias), ptr(running_mean),
                                   ptr(running_var), int(bool(training)), float(eps), float(momentum), ptr(gb), B, 256,
                                   ptr(scsh), ptr(mod), stream())


def synth_input(w, bias, ic, jc, x0, stats, batch):
    """x0[C,HW] = sin(w[:,0]*i + w[:,1]*j + b) and batch-multiplied BN statistics (map3d_layers.py:260-275)."""
    C = w.shape[0]
    with torch.cuda.device_of(x0):
        call("hg_synth_input", ptr(w), ptr(bias), ptr(ic), ptr(jc), C, ic.numel(), jc.numel(), ptr(x0), ptr(stats),
                                   batch, stream())
    return x0


def render_mlp(rec, z_vals, film, wblob, w_sigma, w_rgb, b_feat, heads_b, *, B, R, S, noise=None, noise_std=0.0,
               white_back=False, last_back=False, clamp_mode="relu", passes=3, want_weights=False, raw=False):
    """Fused FiLM-SIREN + ray integration (csrc/render.cu) -> ray_out [B,R,260] (256 feat, 3 rgb, depth)."""
    dev = rec.device
    ray_out = None if raw else torch.empty(B, R, 260, dtype=torch.float32, device=dev)
    raw_out = torch.empty(B, R * S, 260, dtype=torch.float32, device=dev) if raw else None
    weights = torch.empty(B, R * S, dtype=torch.float32, device=dev) if want_weights else None
    if clamp_mode not in ("relu", "softplus"):
        raise RuntimeError("Need to choose clamp mode")          # volume_rendering.py:31
    with torch.cuda.device_of(rec):
        call("hg_render_mlp", ptr(rec), ptr(z_vals), ptr(noise), ptr(film), ptr(wblob), ptr(w_sigma), ptr(w_rgb),
                                  ptr(b_feat), ptr(heads_b), ptr(ray_out), ptr(weights), ptr(raw_out), B, R, S, 256, float(noise_std),
                                  int(bool(white_back)), int(bool(last_back)), int(clamp_mode == "softplus"), passes,
                                  stream())
    return (raw_out if raw else ray_out), weights


def conv2d(x1, wimg, Cout, Nb, *, ksize, H, W, x2=None, up2=False, pre_lrelu=False, bias=None, residual=None,
           res_up2=False, passes=3, out=None):
    """Implicit-GEMM 3x3 / 1x1 convolution (csrc/dconv.cu).  x1 [B,C1,Hs,Ws] (+x2 concat) -> [B,Cout,H,W]."""
    B, C1 = x1.shape[0], x1.shape[1]
    C2 = 0 if x2 is None else x2.shape[1]
    if out is None:
        out = torch.empty(B, Cout, H, W, dtype=torch.float32, device=x1.device)
    with torch.cuda.device_of(x1):
        call("hg_conv2d", ptr(x1), C1, ptr(x2), C2, B, H, W, int(bool(up2)), int(bool(pre_lrelu)), ksize, ptr(wimg), Cout, Nb,
             ptr(bias), ptr(residual), int(bool(res_up2)), ptr(out), passes, stream(),
             tag=f"{C1}+{C2}->{Cout} k{ksize} {H}x{W} B{B}{' up' if up2 else ''}" if TIMING_TAGS else None)
    return out


_CONV_WS = {}


_WGH_WS = {}


def _conv3x3_wgrad_halo(dy, x, passes):
    """3x3 weight gradient on rows of >= 128 pixels (csrc/dconv_wgrad_halo.cu): per (128 output, 64 input)-channel block three
    launches (one filter row of 3 taps each: the accumulators of at most 4 taps fit the registers), the input converted once
    per image row instead of once per tap."""
    B, Cout, H, W = dy.shape
    Cin = x.shape[1]
    dev = dy.device
    ws = _WGH_WS.get(dev)
    if ws is None:
        ws = _WGH_WS[dev] = torch.empty(int(lib().hg_conv3x3_wgrad_halo_workspace_bytes()) // 4, dtype=torch.float32, device=dev)
    dW = torch.empty(Cout, Cin, 9, dtype=torch.float32, device=dev)
    db = torch.empty(Cout, dtype=torch.float32, device=dev)
    groups = ([0, 1, 2], [3, 4, 5], [6, 7, 8])
    for co0 in range(0, Cout, 128):
        nco = min(128, Cout - co0)
        for ci0 in range(0, Cin, 64):
            nci = min(64, Cin - ci0)
            for gi, taps in enumerate(groups):
                n = len(taps)
                tdy = (ctypes.c_int * n)(*[t // 3 - 1 for t in taps])
                tdx = (ctypes.c_int * n)(*[t % 3 - 1 for t in taps])
                dw = torch.empty(n, 128, 64, dtype=torch.float32, device=dev)
                first = ci0 == 0 and gi == 0
                dbt = torch.empty(128, dtype=torch.float32, device=dev) if first else None
                with torch.cuda.device_of(dy):
                    call("hg_conv3x3_wgrad_halo", ptr(dy), ptr(x), ptr(dw), ptr(dbt), ptr(ws), B, H, W, Cout, Cin, co0, nco, ci0, nci,
                         n, ctypes.cast(tdy, c_void_p), ctypes.cast(tdx, c_void_p), passes, stream(),
                         tag=f"{Cin}->{Cout} {H}x{W} B{B}" if TIMING_TAGS else None)
                dW[co0:co0 + nco, ci0:ci0 + nci, taps[0]:taps[-1] + 1] = dw[:, :nco, :nci].permute(1, 2, 0)
                if first:
                    db[co0:co0 + nco] = dbt[:nco]
    return dW.reshape(Cout, Cin, 3, 3), db


def conv2d_wgrad(dy, x, ksize, passes=3):
    """dW [Cout,Cin,k,k], dbias [Cout] of a stride-1 'same' convolution.  3x3 on rows of >= 128 pixels: the haloed kernel
    (csrc/dconv_wgrad_halo.cu); otherwise csrc/dconv_bwd.cu: ONE launch per layer whose grid enumerates the (128 output,
    256 input)-channel chunks and the groups of taps whose accumulators fit the registers (`hg_conv2d_wgrad_layer`; the per-group
    entry point `hg_conv2d_wgrad_taps` stays exported)."""
    B, Cout, H, W = dy.shape
    Cin = x.shape[1]
    dev = dy.device
    dy, x = dy.contiguous(), x.contiguous()
    if ksize == 3 and W % 128 == 0 and os.environ.get("HG3D_WGRAD_HALO", "1") != "0":
        return _conv3x3_wgrad_halo(dy, x, passes)
    need = int(lib().hg_conv2d_wgrad_layer_workspace_bytes(B, H, W, Cout, Cin, ksize))
    ws = _CONV_WS.get(dev)
    if ws is None or ws.numel() * 4 < need:
        ws = _CONV_WS[dev] = torch.empty(max(need, 64 << 20) // 4 + 4, dtype=torch.float32, device=dev)
    dW = torch.empty(Cout, Cin, ksize, ksize, dtype=torch.float32, device=dev)
    db = torch.empty(Cout, dtype=torch.float32, device=dev)
    with torch.cuda.device_of(dy):
        call("hg_conv2d_wgrad_layer", ptr(dy), ptr(x), ptr(dW), ptr(db), ptr(ws), ws.numel() * 4, B, H, W, Cout, Cin, ksize, passes,
             stream(), tag=f"{Cin}->{Cout} k{ksize} {H}x{W} B{B}" if TIMING_TAGS else None)
    return dW, db


def resample2x(x, up, scale):
    """[B,C,H,W] -> 2x2 pooled (up=False: scale * block sum) or nearest up-sampled (up=True: scale * x)."""
    B, C, H, W = x.shape
    y = torch.empty(B, C, H * 2, W * 2, dtype=torch.float32, device=x.device) if up else \
        torch.empty(B, C, H // 2, W // 2, dtype=torch.float32, device=x.device)
    with torch.cuda.device_of(x):
        call("hg_resample2x", ptr(x), ptr(y), B * C, H, W, int(bool(up)), float(scale), stream())
    return y


def pool_add(a, pool_a, b=None, pool_b=False):
    """P_a(a) + P_b(b), P = 2x2 average pooling when flagged."""
    Bn, C, Ha, Wa = a.shape
    H, W = (Ha // 2, Wa // 2) if pool_a else (Ha, Wa)
    out = torch.empty(Bn, C, H, W, dtype=torch.float32, device=a.device)
    with torch.cuda.device_of(a):
        call("hg_pool_add", ptr(a), int(bool(pool_a)), ptr(b), int(bool(pool_b)), ptr(out), Bn * C, H, W, stream())
    return out


def dense(x, w, bias):
    B, K = x.shape
    O = w.shape[0]
    out = torch.empty(B, O, dtype=torch.float32, device=x.device)
    with torch.cuda.device_of(x):
        call("hg_dense", ptr(x), ptr(w), ptr(bias), ptr(out), B, K, O, stream())
    return out


def iso_surface(lattice, level, origin=(0.0, 0.0, 0.0), spacing=1.0):
    """Marching-tetrahedra iso-surface of lattice [Nz,Ny,Nx] fp32 (x fastest) at `level` (csrc/surface.cu; the rule is in
    include/hg3d.h): count + int64 scans, one device-to-host read of the two totals, emit.
    -> (vertices [V,3] fp32, normals [V,3] fp32, faces [F,3] int32); empty tensors when nothing crosses."""
    if lattice.dim() != 3 or lattice.dtype != torch.float32:
        raise RuntimeError(f"hg3d: iso_surface takes a [Nz,Ny,Nx] fp32 lattice (got {tuple(lattice.shape)} {lattice.dtype})")
    nz, ny, nx = lattice.shape
    if min(nz, ny, nx) < 2 or nz * ny * nx > 1 << 30:
        raise RuntimeError(f"hg3d: iso_surface needs >= 2 points per axis and at most 2^30 points (got {nz} x {ny} x {nx})")
    level, spacing = float(level), float(spacing)
    if level != level or not spacing > 0 or len(origin) != 3:
        raise RuntimeError(f"hg3d: iso_surface needs a finite level, a positive spacing and a 3-d origin "
                           f"(got level {level}, spacing {spacing}, origin {origin})")
    dev = lattice.device
    lat = lattice.contiguous()
    nbytes = int(lib().hg_iso_workspace_bytes(nz, ny, nx))
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    totals = torch.empty(2, dtype=torch.int64, device=dev)
    with torch.cuda.device_of(lat):
        call("hg_iso_count", ptr(lat), nz, ny, nx, level, ptr(ws), nbytes, ptr(totals), stream())
        V, F = (int(v) for v in totals.cpu())
        if V >= 1 << 31:
            raise RuntimeError(f"hg3d: iso_surface found {V} vertices; int32 face indices hold fewer than 2^31")
        verts = torch.empty(V, 3, dtype=torch.float32, device=dev)
        normals = torch.empty(V, 3, dtype=torch.float32, device=dev)
        faces = torch.empty(F, 3, dtype=torch.int32, device=dev)
        if V:
            o = [float(v) for v in origin]
            call("hg_iso_emit", ptr(lat), nz, ny, nx, *o, spacing, level, ptr(ws), nbytes, V, ptr(verts), ptr(normals), ptr(faces),
                 stream())
    return verts, normals, faces
