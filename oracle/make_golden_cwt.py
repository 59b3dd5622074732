"""Generate tests/golden/cwt_vectors.{json,npz} from the UNMODIFIED reference -- TEST INFRASTRUCTURE ONLY.

Records what ptwt.cwt computes, so that the suite can check the port and the kernels where the reference is not
installed (continuous wavelets come from oracle/cwt_shim.py when PyWavelets is absent):

* ``signature``: parameter names, kinds and defaults of cwt;
* ``modules``: ``wavefun`` samples ``psi`` of the reference's learnable ``_ShannonWavelet("shan1-1")`` and
  ``_ComplexMorletWavelet("cmor1.5-1.0")`` at precisions 8 and 10 (the GPU tests feed them back as wavelets, with
  the module's grid ``torch.linspace(lower, upper, 2**precision)`` recomputed);
* ``cases``: coefficients and frequencies for mexh, morl, cmor1.5-1.0, shan0.1-0.4 and the two modules; scales
  ``np.arange(1, 16)``, a scalar, ``torch.arange(1, 15)``, geometric float scales including s < 1 and a float32
  array; lengths 1, 2, 31, 32, 200 and 1000 (filters longer than the signal included); inputs ``[n]``, ``[3, n]``
  and ``[2, 3, n]``; float32 and float64; precision 8, 10 and 12 and a non-default ``sampling_period``.  The input
  of one (shape) is stored once in float64 (``x_<shape>``); float32 cases round it;
* ``grads``: the input gradient of the loss ``sum(loss_weights(coef.shape) * coef)`` (real and imaginary parts
  weighted separately), for a real and a complex wavelet, float64 and float32; the weights are a closed form, not
  stored;

The coefficients are float64 / complex128 random-input values that do not compress, so the cases are sized to keep
the archive well under 1 MB: long signals and many scales are compared with the port in the GPU tests instead.
* ``errors``: the exception type of each error case.

    python -m oracle.make_golden_cwt
"""
from __future__ import annotations

import inspect
import json
from pathlib import Path

import numpy as np
import torch

from oracle.cwt_fixture import loss_weights
from oracle.cwt_shim import import_reference

OUT = Path(__file__).resolve().parent.parent / "tests" / "golden"
NAMES = ("mexh", "morl", "cmor1.5-1.0", "shan0.1-0.4")
MODULES = {"shan1-1": "_ShannonWavelet", "cmor1.5-1.0": "_ComplexMorletWavelet"}
PRECISIONS = (8, 10, 12)
MODULE_PRECISIONS = (8, 10)

SCALES = {
    "arange": np.arange(1, 16),
    "scalar": 5.0,
    "torch": torch.arange(1, 15),
    "geom": np.geomspace(0.25, 48.0, 7),
    "f32": np.array([0.75, 1.5, 2.25, 6.5, 11.0], dtype=np.float32),
}


def scales_to_store(spec: str) -> np.ndarray:
    s = SCALES[spec]
    return s.numpy() if isinstance(s, torch.Tensor) else np.asarray(s)


def case_list():
    """(wavelet, scales, shape, dtype, precision, sampling_period)."""
    cases = []
    for w in NAMES + tuple("module:" + m for m in MODULES):
        prec = 10 if w.startswith("module:") else 12
        cases.append((w, "arange", (31,), "float64", prec, 1.0))            # K up to 241 > n
        cases.append((w, "geom", (3, 32), "float64", prec, 1.0))
        cases.append((w, "f32", (200,), "float32", prec, 1.0))
        cases.append((w, "scalar", (2, 3, 31), "float64", 10 if prec == 12 else 8, 0.25))
    for w in ("morl", "cmor1.5-1.0"):
        for n in (1, 2):
            cases.append((w, "arange", (3, n), "float64", 12, 1.0))
            cases.append((w, "geom", (n,), "float32", 12, 1.0))
    cases.append(("morl", "torch", (2, 3, 32), "float32", 12, 1.0))
    cases.append(("cmor1.5-1.0", "torch", (3, 32), "float32", 12, 1.0))
    cases.append(("morl", "geom", (1000,), "float64", 12, 1.0))
    cases.append(("shan0.1-0.4", "scalar", (1000,), "float32", 12, 1.0))
    for prec in PRECISIONS:
        cases.append(("mexh", "arange", (32,), "float64", prec, 4 * np.pi / 800))
        cases.append(("shan0.1-0.4", "torch", (32,), "float32", prec, 1.0))
    cases.append(("module:shan1-1", "torch", (2, 3, 32), "float32", 8, 0.5))
    return cases


def make_wavelet(ptwt, spec: str):
    if spec.startswith("module:"):
        name = spec.split(":", 1)[1]
        return getattr(ptwt.continuous_transform, MODULES[name])(name)
    return spec


def main() -> None:
    ptwt = import_reference()
    g = torch.Generator().manual_seed(20261016)
    meta: dict = {"signature": [], "modules": {}, "cases": [], "grads": [], "errors": []}
    arrays: dict = {}
    for p in inspect.signature(ptwt.cwt).parameters.values():
        meta["signature"].append({"name": p.name, "kind": p.kind.name,
                                  "default": None if p.default is inspect.Parameter.empty else repr(p.default)})
    with torch.no_grad():
        for name, cls in MODULES.items():
            mod = getattr(ptwt.continuous_transform, cls)(name)
            meta["modules"][name] = {"class": cls, "complex_cwt": bool(mod.complex_cwt),
                                     "bounds": [float(mod.lower_bound), float(mod.upper_bound)]}
            for prec in MODULE_PRECISIONS:
                psi, grid = mod.wavefun(prec)
                assert torch.equal(grid, torch.linspace(mod.lower_bound, mod.upper_bound, 2 ** prec,
                                                        dtype=torch.float64))
                arrays[f"module_{name}_p{prec}_psi"] = psi.numpy()
    for spec in SCALES:
        arrays[f"scales_{spec}"] = scales_to_store(spec)

    inputs: dict = {}

    def input_for(shape):
        key = "x_" + "x".join(map(str, shape))
        if key not in inputs:
            inputs[key] = torch.randn(shape, generator=g, dtype=torch.float64)
            arrays[key] = inputs[key].numpy()
        return key, inputs[key]

    for i, (w, sc, shape, dt, prec, sp) in enumerate(case_list()):
        xkey, x = input_for(shape)
        x = x.to(getattr(torch, dt))
        with torch.no_grad():
            coef, freqs = ptwt.cwt(x, SCALES[sc], make_wavelet(ptwt, w), sampling_period=sp, precision=prec)
        cid = f"c{i}"
        arrays[cid + "_coef"] = coef.numpy()
        arrays[cid + "_freqs"] = np.asarray(freqs)
        meta["cases"].append({"id": cid, "wavelet": w, "scales": sc, "shape": list(shape), "dtype": dt,
                              "precision": prec, "sampling_period": sp, "x": xkey,
                              "coef_dtype": str(coef.dtype).replace("torch.", ""), "freqs_dtype": str(freqs.dtype)})

    for w in ("morl", "cmor1.5-1.0"):
        for dt in ("float64", "float32"):
            shape = (2, 100)
            xkey, x0 = input_for(shape)
            x = x0.detach().to(getattr(torch, dt)).clone().requires_grad_(True)
            coef, _ = ptwt.cwt(x, np.arange(1, 8), w)
            key = f"g_{w}_{dt}"
            if coef.is_complex():
                loss = (torch.view_as_real(coef) * loss_weights(coef.shape + (2,))).sum()
            else:
                loss = (coef * loss_weights(coef.shape)).sum()
            loss.backward()
            arrays[key + "_grad"] = x.grad.numpy()
            meta["grads"].append({"id": key, "wavelet": w, "dtype": dt, "x": xkey, "scales": "arange1_8",
                                  "complex": bool(coef.is_complex())})

    x = torch.randn(16, generator=g, dtype=torch.float64)
    for label, scales in (("zero", np.array([0.0])), ("negative", np.array([-1.0])), ("tiny", np.array([0.01]))):
        try:
            ptwt.cwt(x, scales, "morl")
            kind = None
        except Exception as e:  # noqa: BLE001
            kind = type(e).__name__
        meta["errors"].append({"case": label, "scales": scales.tolist(), "raises": kind})

    OUT.mkdir(parents=True, exist_ok=True)
    np.savez_compressed(OUT / "cwt_vectors.npz", **arrays)
    (OUT / "cwt_vectors.json").write_text(json.dumps(meta, indent=1) + "\n")
    size = (OUT / "cwt_vectors.npz").stat().st_size
    print(f"{len(meta['cases'])} cases, {len(meta['grads'])} grads, npz {size / 1e6:.2f} MB")


if __name__ == "__main__":
    main()
