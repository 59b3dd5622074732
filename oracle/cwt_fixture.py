"""Reading tests/golden/cwt_vectors.{json,npz} back into cwt arguments -- TEST INFRASTRUCTURE ONLY."""
from __future__ import annotations

import json
from functools import lru_cache
from pathlib import Path

import numpy as np
import torch

GOLDEN = Path(__file__).resolve().parent.parent / "tests" / "golden"


@lru_cache(maxsize=1)
def load():
    meta = json.loads((GOLDEN / "cwt_vectors.json").read_text())
    with np.load(GOLDEN / "cwt_vectors.npz") as z:
        arrays = {k: z[k] for k in z.files}
    return meta, arrays


class StoredWavelet(torch.nn.Module):
    """Plays the reference's learnable wavelet module whose ``wavefun`` samples the fixture stores: a complex
    ``nn.Module`` wavelet (so its ``int_psi`` is conjugated) without parameters."""

    complex_cwt = True

    def __init__(self, name: str):
        super().__init__()
        meta, _ = load()
        self.name = name
        self.lower_bound, self.upper_bound = meta["modules"][name]["bounds"]

    def wavefun(self, precision: int, dtype: torch.dtype = torch.float64):
        _, arrays = load()
        psi = torch.from_numpy(arrays[f"module_{self.name}_p{precision}_psi"])
        # the module's own grid (the generator checks that it is exactly this)
        grid = torch.linspace(self.lower_bound, self.upper_bound, 2 ** precision, dtype=torch.float64)
        return psi, grid


def loss_weights(shape) -> torch.Tensor:
    """Fixed float64 weights of the gradient cases (a closed form, so nothing is stored); a complex coefficient's
    real and imaginary parts are weighted by ``loss_weights(shape + (2,))`` through ``torch.view_as_real``."""
    k = torch.arange(int(np.prod(shape)), dtype=torch.float64)
    return torch.sin(0.731 * k + 0.3).reshape(tuple(shape))


def wavelet(case: dict):
    w = case["wavelet"]
    return StoredWavelet(w.split(":", 1)[1]) if w.startswith("module:") else w


def scales(case: dict):
    _, arrays = load()
    s = arrays["scales_" + case["scales"]]
    if case["scales"] == "scalar":
        return float(s)
    if case["scales"] == "torch":
        return torch.from_numpy(s)
    return s


def data(case: dict) -> torch.Tensor:
    _, arrays = load()
    return torch.from_numpy(arrays[case["x"]]).to(getattr(torch, case["dtype"]))
