"""Generate tests/golden/reference_api.* from the UNMODIFIED reference -- TEST INFRASTRUCTURE ONLY.

The transform vectors of make_golden.py pin the oracle port; this file stores everything else the tests compare
with the reference itself, so that the suite runs where the reference is not installed:

* ``port_cases``: the oracle port must equal the reference bit for bit on the conv path (every mode, float32 and
  float64) and to round-off on the matrix classes;
* ``fs_cases``: the reference's fswavedec2 / fswavedec3 bands and fswaverec2 (the claim behind ``separable.py``);
* ``matrix_warnings``: the reference's stderr warning of the separable matrix level walk;
* ``signatures``: parameter names, kinds and defaults of every public reference callable;
* ``packet_orders``: WaveletPacket / WaveletPacket2D key orders;
* ``install``: wavedec2 of the reference on the input of the install() round trip;
* ``learnable``: the loss and the gradients the reference computes through learnable ProductFilter taps.

    python -m oracle.make_golden_api
"""
from __future__ import annotations

import contextlib
import inspect
import io
import json
from pathlib import Path

import numpy as np
import torch

from oracle.ref_import import import_reference

OUT = Path(__file__).resolve().parent.parent / "tests" / "golden"
MODES = ("zero", "constant", "reflect", "periodic", "symmetric")


def flatten(coeffs):
    """Coefficient pytree -> flat list (order of tests/conftest.py flatten_coeffs)."""
    out = []
    for el in coeffs:
        if isinstance(el, torch.Tensor):
            out.append(el)
        elif isinstance(el, dict):
            out.extend(el[k] for k in ("aad", "ada", "add", "daa", "dad", "dda", "ddd"))
        else:
            out.extend(el)
    return out


def run_case(mod, case, x):
    """(coefficients, reconstruction) of one port case with module ``mod`` (the reference or the port)."""
    fn, wav, level, kw = case["fn"], case["wavelet"], case["level"], dict(case["kw"])
    if fn in ("wavedec", "wavedec2", "wavedec3"):
        c = getattr(mod, fn)(x, wav, level=level, **kw)
        return c, getattr(mod, fn.replace("dec", "rec"))(c, wav)
    c = getattr(mod, fn)(wav, level, **kw)(x)
    return c, getattr(mod, fn.replace("dec", "rec"))(wav)(c)


def port_cases():
    g = torch.Generator().manual_seed(7)
    cases = []
    for mode in MODES:
        x = torch.randn(1, 9, 10, generator=g, dtype=torch.float64)
        x3 = torch.randn(1, 5, 6, 7, generator=g, dtype=torch.float64)
        for dtype in ("float64", "float32"):
            for fn, wav, level, data in (("wavedec", "db3", 2, x), ("wavedec2", "db2", 2, x), ("wavedec3", "db2", 1, x3)):
                cases.append(dict(fn=fn, wavelet=wav, level=level, kw={"mode": mode}, tol=0.0, rec_tol=0.0,
                                  dtype=dtype, x=data.to(getattr(torch, dtype))))
    cases.append(dict(fn="MatrixWavedec", wavelet="db4", level=3, kw={}, tol=1e-13, rec_tol=1e-12, dtype="float64",
                      x=torch.randn(2, 64, generator=g, dtype=torch.float64)))
    for odd_mode in MODES:
        cases.append(dict(fn="MatrixWavedec2", wavelet="db3", level=2, kw={"odd_coeff_padding_mode": odd_mode},
                          tol=1e-12, rec_tol=1e-11, dtype="float64",
                          x=torch.randn(1, 15, 18, generator=g, dtype=torch.float64)))
        cases.append(dict(fn="MatrixWavedec3", wavelet="db2", level=2, kw={"odd_coeff_padding_mode": odd_mode},
                          tol=1e-12, rec_tol=1e-11, dtype="float64",
                          x=torch.randn(1, 9, 8, 7, generator=g, dtype=torch.float64)))
    return cases


def params(fn):
    return [[n, p.kind.name, repr(p.default)] for n, p in inspect.signature(fn).parameters.items() if n != "self"]


def main() -> None:
    ptwt = import_reference()
    arrays, man = {}, {"generated_by": "oracle/make_golden_api.py", "torch": torch.__version__}

    man["port_cases"] = []
    for i, case in enumerate(port_cases()):
        key = f"port{i}"
        x = case.pop("x")
        c, rec = run_case(ptwt, case, x)
        flat = flatten(c)
        if case["dtype"] == "float64":
            arrays[f"{key}_x"] = x.numpy()
        else:                                           # the float64 input of the same mode, rounded
            case["x_from"] = f"port{i - 3}"
        arrays[f"{key}_o"] = np.concatenate([t.reshape(-1).numpy() for t in flat] + [rec.reshape(-1).numpy()])
        man["port_cases"].append(dict(case, key=key, shapes=[list(t.shape) for t in flat], rec_shape=list(rec.shape)))

    g = torch.Generator().manual_seed(9)
    x = torch.randn(1, 17, 20, generator=g, dtype=torch.float64)
    arrays["fs2_x"] = x.numpy()
    man["fs_cases"] = []
    for mode in ("zero", "reflect", "constant", "periodic"):
        fs = ptwt.fswavedec2(x, "db2", mode=mode, level=2)
        key = f"fs2_{mode}"
        arrays[f"{key}_a"] = fs[0].numpy()
        for lv, d in enumerate(fs[1:]):
            for k, v in d.items():
                arrays[f"{key}_d{lv}_{k}"] = v.contiguous().numpy()
        man["fs_cases"].append({"key": key, "mode": mode, "keys": [list(d.keys()) for d in fs[1:]]})
        arrays[f"{key}_rec"] = ptwt.fswaverec2(fs, "db2").numpy()
    x3 = torch.randn(1, 8, 9, 10, generator=g, dtype=torch.float64)
    fs = ptwt.fswavedec3(x3, "db2", mode="zero", level=1)
    arrays["fs3_x"] = x3.numpy()
    for k, v in fs[1].items():
        arrays[f"fs3_d0_{k}"] = v.contiguous().numpy()
    man["fs3_keys"] = list(fs[1].keys())

    warnings = {}
    for name, cls, wav, shape in (("matrix3_db2_L3_12x9x16", ptwt.MatrixWavedec3, "db2", (12, 9, 16)),
                                  ("matrix2_db3_L3_20x12", ptwt.MatrixWavedec2, "db3", (20, 12))):
        buf = io.StringIO()
        with contextlib.redirect_stderr(buf):
            cls(wav, 3)(torch.randn(shape, dtype=torch.float64))
        warnings[name] = buf.getvalue()
    man["matrix_warnings"] = warnings

    sig = {}
    for name in ("wavedec", "waverec", "wavedec2", "waverec2", "wavedec3", "waverec3", "fswavedec2", "fswavedec3",
                 "fswaverec2", "fswaverec3"):
        sig[name] = params(getattr(ptwt, name))
    for name in ("MatrixWavedec", "MatrixWaverec", "MatrixWavedec2", "MatrixWaverec2", "MatrixWavedec3",
                 "MatrixWaverec3", "WaveletPacket", "WaveletPacket2D"):
        sig[name] = params(inspect.unwrap(getattr(ptwt, name).__init__))
    man["signatures"] = sig

    man["packet_orders"] = {str(lev): {"level": ptwt.WaveletPacket.get_level(lev),
                                       "level_natural": ptwt.WaveletPacket.get_level(lev, "natural"),
                                       "freq_2d": ptwt.WaveletPacket2D.get_freq_order(lev),
                                       "natural_2d": ptwt.WaveletPacket2D.get_natural_order(lev)}
                            for lev in (0, 1, 2, 3)}

    g = torch.Generator().manual_seed(11)
    x = torch.randn(1, 2, 32, 24, generator=g)
    arrays["install_x"] = x.numpy()
    flat = flatten(ptwt.wavedec2(x, "db2", level=2))
    for j, t in enumerate(flat):
        arrays[f"install_o{j}"] = t.contiguous().numpy()
    man["install_n_out"] = len(flat)

    from ptwt.wavelets_learnable import ProductFilter

    from pytorch_wavelet_toolbox_b200 import _wavelets
    from pytorch_wavelet_toolbox_b200.constants import WaveletTensorTuple

    fb = WaveletTensorTuple.from_wavelet(_wavelets.as_wavelet("db3"), torch.float64)
    wav = ProductFilter(*[t.clone() for t in fb])
    g = torch.Generator().manual_seed(3)
    x = torch.randn(2, 96, generator=g, dtype=torch.float64)
    w = torch.randn(2, 96, generator=g, dtype=torch.float64)
    xr = x.clone().requires_grad_(True)
    c = ptwt.wavedec(xr, wav, level=3, mode="reflect")
    rec = ptwt.waverec(c, wav)[..., :96]
    loss = sum((t * t).sum() for t in c) + (rec * w).sum()
    loss.backward()
    arrays["learn_x"], arrays["learn_w"], arrays["learn_grad_x"] = x.numpy(), w.numpy(), xr.grad.numpy()
    for name in ("dec_lo", "dec_hi", "rec_lo", "rec_hi"):
        arrays[f"learn_grad_{name}"] = getattr(wav, name).grad.numpy()
    man["learnable"] = {"wavelet": "db3", "level": 3, "mode": "reflect", "loss": float(loss.detach())}

    np.savez_compressed(OUT / "reference_api.npz", **arrays)
    (OUT / "reference_api.json").write_text(json.dumps(man, indent=1))
    print("wrote", OUT / "reference_api.npz", sum(v.nbytes for v in arrays.values()), "bytes raw")


if __name__ == "__main__":
    main()
