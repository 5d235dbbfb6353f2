"""Rebuild the exact inputs of a golden fixture from its recipe (tests/golden/manifest.json)."""
import importlib
import json
import os

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden")


def manifest():
    with open(os.path.join(GOLD, "manifest.json")) as f:
        return json.load(f)


def load(name):
    return {k: torch.from_numpy(v) for k, v in np.load(os.path.join(GOLD, name + ".npz")).items()}


def generator_case(name):
    """-> cfg, params, cond, z, (u, noise), golden outputs."""
    pkg = importlib.import_module("3dhumangan_b200")
    from oracle import port
    m = manifest()[name]
    base, over, pseed, sg, sb, B, noise_std = m["recipe"]
    cfg = pkg.configs.baseline_config(base)
    cfg.update(over)
    cfg["nerf_noise"] = noise_std
    params = port.init_generator_params(cfg, seed=pseed, sigma_gain=sg, sigma_bias=sb)
    cond = pkg.synthetic.make_conditions(B, seed=11 + pseed)
    z = torch.randn(B, cfg["latent_dim"], generator=torch.Generator().manual_seed(100 + pseed))
    torch.manual_seed(m["rng_seed"])
    u, noise = pkg.rng.draw_render_noise(B, cfg["render_width"] * cfg["render_height"], cfg["num_steps"], "cpu",
                                         cfg["sample_dist"])
    return cfg, params, cond, z, (u, noise), load(name)


def discriminator_case(name):
    pkg = importlib.import_module("3dhumangan_b200")
    from oracle import port
    over, pseed, B = manifest()[name]["recipe"]
    cfg = pkg.configs.baseline_config("C2")
    cfg.update(over)
    params = port.init_discriminator_params(cfg, seed=pseed)
    img = torch.randn(B, 3, cfg["gen_height"], cfg["gen_width"], generator=torch.Generator().manual_seed(pseed)).clamp(-1, 1)
    return cfg, params, img, load(name)


def rel_l2(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


# ---- results of the reference's own code, recorded once by tests/golden/make_golden_trainer.py so that the tests that pin
# this package against the reference need nothing outside the repository
REFERENCE_RESULTS = os.path.join(GOLD, "reference_results.npz")
RECORDING = None      # {key: value} while make_golden_trainer.py runs those tests against a reference checkout
_recorded = None


class RecordedClass(str):
    """A class of the reference, recorded by its name: equal to any class (or string) of that name."""

    def __new__(cls, name):
        obj = str.__new__(cls, name)
        obj.__name__ = name
        return obj

    def __eq__(self, other):
        return str.__eq__(self, other if isinstance(other, str) else getattr(other, "__name__", None))

    __hash__ = str.__hash__


def _encode(v, arrays):
    if torch.is_tensor(v):
        arrays[f"a{len(arrays)}"] = v.detach().numpy()
        return {"tensor": f"a{len(arrays) - 1}"}
    if isinstance(v, (tuple, list)):
        return {"tuple" if isinstance(v, tuple) else "list": [_encode(x, arrays) for x in v]}
    if isinstance(v, dict):
        return {"dict": [[_encode(k, arrays), _encode(x, arrays)] for k, x in v.items()]}
    if isinstance(v, type):
        return {"class": v.__name__}
    assert v is None or isinstance(v, (bool, int, float, str)), type(v)
    return {"value": v}


def _decode(v, arrays):
    (kind, x), = v.items()
    if kind == "tensor":
        return torch.from_numpy(arrays[x])
    if kind in ("tuple", "list"):
        items = [_decode(i, arrays) for i in x]
        return tuple(items) if kind == "tuple" else items
    if kind == "dict":
        return {_decode(k, arrays): _decode(i, arrays) for k, i in x}
    return RecordedClass(x) if kind == "class" else x


def reference_result(key, compute):
    """What the reference's own code `compute()` returned for `key`: computed while recording, read back otherwise."""
    global _recorded
    if RECORDING is not None:
        RECORDING[key] = value = compute()
        return value
    if _recorded is None:
        raw = np.load(REFERENCE_RESULTS)
        _recorded = json.loads(str(raw["index"])), {k: raw[k] for k in raw.files if k != "index"}
    index, arrays = _recorded
    return _decode(index[key], arrays)


def save_reference_results():
    arrays = {}
    index = {k: _encode(v, arrays) for k, v in RECORDING.items()}
    np.savez_compressed(REFERENCE_RESULTS, index=np.array(json.dumps(index, sort_keys=True)), **arrays)
