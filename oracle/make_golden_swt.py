"""Generate tests/golden/swt_vectors.{json,npz} from the UNMODIFIED reference -- TEST INFRASTRUCTURE ONLY.

Records what ptwt.swt / ptwt.iswt compute, so that the suite can check the port and the kernels where the reference
is not installed:

* ``signatures``: parameter names, kinds and defaults of swt and iswt;
* ``cases``: coefficients and reconstructions for six named wavelets and one custom non-orthogonal filter bank
  (a 4-tuple of tensors), float64 (float32 for F32_WAVELETS), lengths 1 .. 1000, levels None / 1 / swt_max_level / explicit levels
  past it (``quirk``: the level's extension is not periodic), inputs of 1, 2 and 4 dims and a non-default axis; the
  input of the cases of one length is stored once (``x<n>``, float64; the float32 cases round it);
* ``grads``: the input gradient of a fixed weighted loss through swt and through iswt;
* ``errors``: the exception type of each error case.

    python -m oracle.make_golden_swt
"""
from __future__ import annotations

import inspect
import json
from pathlib import Path

import numpy as np
import torch

from oracle.ref_import import import_reference
from oracle.swt_closed_form import periodic
from oracle.swt_port import extension_index

OUT = Path(__file__).resolve().parent.parent / "tests" / "golden"
WAVELETS = ("haar", "db2", "db3", "db4", "sym5", "db8", "custom")
LENGTHS = (1, 14, 37, 48, 64, 96, 1000)
#: the fixtures stay small: from LONG on one filter bank and no level 1; swt_max_level passed explicitly (the same
#: numbers as level=None) for one filter bank only.  The GPU tests compare long signals with the port.
LONG = 1000
LONG_WAVELETS = ("db4",)
EXPLICIT_MAX_WAVELETS = ("custom",)
#: float32 cases for three filter banks (float64 for all seven)
F32_WAVELETS = ("haar", "db4", "custom")


def custom_bank(dtype: torch.dtype):
    """A biorthogonal-style 4-tap bank that is not orthogonal (no name, passed as a 4-tuple of tensors)."""
    dec_lo = torch.tensor([-0.125, 0.375, 0.875, -0.125], dtype=torch.float64)
    dec_hi = torch.tensor([0.25, -0.75, 0.75, -0.25], dtype=torch.float64)
    rec_lo = torch.tensor([0.25, 0.75, 0.75, 0.25], dtype=torch.float64)
    rec_hi = torch.tensor([-0.125, -0.375, 0.875, 0.125], dtype=torch.float64)
    return tuple(t.to(dtype) for t in (dec_lo, dec_hi, rec_lo, rec_hi))


def wavelet_arg(name: str, dtype: torch.dtype):
    return custom_bank(dtype) if name == "custom" else name


def filt_len(ptwt, name: str) -> int:
    return 4 if name == "custom" else len(ptwt._util._as_wavelet(name))


def is_quirk(n: int, L: int, level: int) -> bool:
    """Whether any level up to ``level`` extends (analysis or synthesis) non-periodically."""
    for j in range(1, level + 1):
        d = 2 ** (j - 1)
        for pl, pr in ((d * (L // 2 - 1), d * (L // 2)), (d * (L // 2), d * (L // 2 - 1))):
            if max(pl, pr) > n and not np.array_equal(extension_index(n, pl, pr).numpy(), periodic(n, pl, pr)):
                return True
    return False


def levels_for(n: int, name: str, L: int, max_level: int):
    """None (= swt_max_level), 1, swt_max_level passed explicitly, and one level past it (the first one that hits
    the quirk, if any), thinned as LONG and EXPLICIT_MAX_WAVELETS say."""
    out = [None]
    if max_level != 1 and n < LONG:
        out.append(1)
    if max_level > 1 and n < LONG and name in EXPLICIT_MAX_WAVELETS:
        out.append(max_level)
    deep = [lv for lv in range(max(max_level, 1) + 1, max(max_level, 1) + 5) if is_quirk(n, L, lv)]
    out.append(deep[0] if deep else max(max_level, 1) + 1)
    return out


def params(fn):
    return [[n, p.kind.name, repr(p.default)] for n, p in inspect.signature(fn).parameters.items()]


def err_type(fn) -> str:
    try:
        fn()
    except Exception as ex:  # noqa: BLE001
        return type(ex).__name__
    return "none"


def main() -> None:
    ptwt = import_reference()
    import pywt

    arrays, man = {}, {"generated_by": "oracle/make_golden_swt.py", "torch": torch.__version__}
    man["signatures"] = {"swt": params(ptwt.swt), "iswt": params(ptwt.iswt)}
    g = torch.Generator().manual_seed(21)
    cases = []
    for n in LENGTHS:
        # one float64 input per length, shared by every case of that length; float32 cases round it
        x64 = torch.randn(1, n, generator=g, dtype=torch.float64)
        arrays[f"x{n}"] = x64.numpy()
        for name in WAVELETS if n < LONG else LONG_WAVELETS:
            L = filt_len(ptwt, name)
            for level in levels_for(n, name, L, pywt.swt_max_level(n)):
                for dtype in ("float64", "float32") if name in F32_WAVELETS else ("float64",):
                    key = f"c{len(cases)}"
                    x = x64.to(getattr(torch, dtype))
                    wav = wavelet_arg(name, x.dtype)
                    c = ptwt.swt(x, wav, level)
                    rec = ptwt.iswt(c, wav)
                    arrays[f"{key}_c"] = torch.stack(c, 0).numpy()
                    arrays[f"{key}_r"] = rec.numpy()
                    lv = pywt.swt_max_level(n) if level is None else level
                    cases.append(dict(key=key, x=f"x{n}", n=n, wavelet=name, level=level, dtype=dtype, filt_len=L,
                                      quirk=bool(lv > 0 and is_quirk(n, L, lv)), shape=list(x64.shape), axis=None))
    # leading dims and a non-default axis
    for shape, axis, level in (((48,), None, 3), ((2, 3, 2, 64), None, 4), ((64, 3), 0, 3), ((2, 96, 3), 1, 5),
                               ((2, 3, 14), -1, 3)):
        key = f"c{len(cases)}"
        x = torch.randn(*shape, generator=g, dtype=torch.float64)
        c = ptwt.swt(x, "db3", level, axis=axis)
        rec = ptwt.iswt(c, "db3", axis=axis)
        arrays[f"{key}_x"] = x.numpy()
        arrays[f"{key}_c"] = torch.stack(c, 0).numpy()
        arrays[f"{key}_r"] = rec.numpy()
        n = shape[axis if axis is not None else -1]
        cases.append(dict(key=key, x=f"{key}_x", n=n, wavelet="db3", level=level, dtype="float64", filt_len=6,
                          quirk=is_quirk(n, 6, level), shape=list(shape), axis=axis))
    man["cases"] = cases

    grads = []
    for n, name, level in ((64, "db4", 3), (14, "db4", 3), (96, "sym5", None), (37, "custom", 2)):
        key = f"g{len(grads)}"
        x = torch.randn(3, n, generator=g, dtype=torch.float64)
        wav = wavelet_arg(name, torch.float64)
        lv = pywt.swt_max_level(n) if level is None else level
        w = torch.randn(lv + 1, 3, n, generator=g, dtype=torch.float64)
        xr = x.clone().requires_grad_(True)
        c = ptwt.swt(xr, wav, level)
        sum((wk * ck).sum() for wk, ck in zip(w, c)).backward()
        cin = [t.detach().clone().requires_grad_(True) for t in ptwt.swt(x, wav, level)]
        wy = torch.randn(3, n, generator=g, dtype=torch.float64)
        (ptwt.iswt(cin, wav) * wy).sum().backward()
        arrays[f"{key}_x"], arrays[f"{key}_w"], arrays[f"{key}_wy"] = x.numpy(), w.numpy(), wy.numpy()
        arrays[f"{key}_gx"] = xr.grad.numpy()
        arrays[f"{key}_gc"] = torch.stack([t.grad for t in cin], 0).numpy()
        grads.append(dict(key=key, n=n, wavelet=name, level=level))
    man["grads"] = grads

    x = torch.randn(2, 16, generator=g)
    c = ptwt.swt(x, "db2", 2)
    man["errors"] = {
        "swt_int": err_type(lambda: ptwt.swt(x.to(torch.int32), "db2", 1)),
        "swt_half": err_type(lambda: ptwt.swt(x.half(), "db2", 1)),
        "swt_axis_out_of_range": err_type(lambda: ptwt.swt(x, "db2", 1, axis=5)),
        "swt_axis_tuple": err_type(lambda: ptwt.swt(x, "db2", 1, axis=(0, 1))),
        "iswt_int": err_type(lambda: ptwt.iswt([t.to(torch.int32) for t in c], "db2")),
        "iswt_axis_out_of_range": err_type(lambda: ptwt.iswt(c, "db2", axis=5)),
        "iswt_mixed_dtype": err_type(lambda: ptwt.iswt([c[0], c[1].double(), c[2]], "db2")),
        "iswt_unequal_length": err_type(lambda: ptwt.iswt([c[0], c[1][..., :8], c[2]], "db2")),
        "iswt_unequal_batch": err_type(lambda: ptwt.iswt([c[0], c[1][:1], c[2]], "db2")),
    }
    man["swt_max_level"] = {str(n): pywt.swt_max_level(n) for n in (1, 2, 3, 14, 37, 48, 64, 96, 1000, 1 << 20)}

    np.savez_compressed(OUT / "swt_vectors.npz", **arrays)
    (OUT / "swt_vectors.json").write_text(json.dumps(man, indent=1))
    print("wrote", OUT / "swt_vectors.npz", len(cases), "cases", sum(v.nbytes for v in arrays.values()), "bytes raw")


if __name__ == "__main__":
    main()
