"""Generate tests/golden/bank_vectors.{json,npz} from the UNMODIFIED reference -- TEST INFRASTRUCTURE ONLY.

Records what ptwt computes with filter banks that are not orthogonal (tests/filter_banks.py: bior2.2, CDF 9/7 and two
unstructured random banks), so that the suite can pin the oracle port and check the kernels where the reference is
not installed.  Orthogonal banks cannot tell ``rec`` from reversed ``dec`` or ``dec_hi`` from the alternating flip of
``dec_lo``; these can.

* ``banks``: the four filters of every bank (``<bank>_taps``, [4, L] float64) -- the fixture does not depend on
  tests/filter_banks.py staying the same;
* ``cases``: wavedec / waverec, wavedec2 / waverec2 and wavedec3 / waverec3 for every bank in all five modes, in
  float64 (1-D and 2-D: level None) and float32 (an explicit level), odd extents, and one non-default axis / axes per
  dimension.  3-D reflect and periodic cases need volumes larger than the filter: those run one level, in one dtype
  per bank.  ``<key>_x`` is the input; ``<key>_o`` holds the coefficients in conftest.flatten_coeffs order and then
  the reconstruction, flattened and concatenated (``shapes`` in the manifest);
* ``packets``: one WaveletPacket and one WaveletPacket2D, every node of the full tree (sorted keys) and the
  reconstruction, concatenated the same way;
* ``grads``: per dimension, the gradient of a fixed weighted loss of the coefficients and of the reconstruction with
  respect to the data and to all four filters (a 4-tuple of float64 tensors): the weights ``<key>_w`` (coefficients,
  then reconstruction, concatenated), ``<key>_gx`` and ``<key>_gtaps`` ([4, L]).

    python -m oracle.make_golden_banks
"""
from __future__ import annotations

import json
import sys
from pathlib import Path

import numpy as np
import torch

from oracle.ref_import import import_reference

ROOT = Path(__file__).resolve().parent.parent
OUT = ROOT / "tests" / "golden"
MODES = ("zero", "constant", "reflect", "periodic", "symmetric")
BANKS = ("bior2.2", "cdf9/7", "unstructured6", "unstructured8")
#: shapes (batch first) and the explicit level of the float32 cases; float64 cases use level None (1-D, 2-D) or 1 (3-D:
#: the default level of a volume this small is 0 for the longer banks).  3-D levels stay at 1 because every level
#: grows a volume this small (the gradient case runs two).
SHAPES = {1: (2, 53), 2: (1, 19, 21), 3: (1, 3, 4, 5)}
SHAPES_F32 = {1: (2, 53), 2: (1, 13, 15), 3: (1, 3, 4, 5)}
LEVEL_F32 = {1: 3, 2: 2, 3: 1}


#: modes whose padding must be shorter (reflect) or not longer (periodic) than the extent it pads
NEEDS_EXTENT = ("reflect", "periodic")


def shape_3d_long_pad(filt_len: int) -> tuple:
    """A level pads L - 2 (+1 on odd extents) samples: the smallest volume whose every extent allows one level in
    reflect and periodic mode (both dtypes run one level there)."""
    return (1, filt_len, filt_len + 1, filt_len + 2)


#: one non-default axis / axes per dimension: (shape, axes, level)
AXES_CASES = {1: ((29, 3), 0, 2), 2: ((11, 2, 13), (0, 2), 2), 3: ((7, 1, 6, 5), (0, 2, 3), 1)}
GRAD_CASES = {1: ("unstructured8", "reflect", (2, 41), 3), 2: ("unstructured6", "symmetric", (1, 17, 19), 2),
              3: ("unstructured8", "zero", (1, 7, 6, 9), 2)}
PACKETS = ((1, "unstructured8", "reflect", (2, 40), 2), (2, "cdf9/7", "periodic", (1, 18, 20), 2))


def banks() -> dict:
    sys.path.insert(0, str(ROOT / "tests"))
    import filter_banks as FB

    return {"bior2.2": FB.bior22(), "cdf9/7": FB.cdf97(), "unstructured6": FB.unstructured(6),
            "unstructured8": FB.unstructured(8)}


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


def key_of(bank: str) -> str:
    return bank.replace("/", "_").replace(".", "")


def transforms(ptwt, ndim: int):
    return {1: (ptwt.wavedec, ptwt.waverec, "axis"), 2: (ptwt.wavedec2, ptwt.waverec2, "axes"),
            3: (ptwt.wavedec3, ptwt.waverec3, "axes")}[ndim]


def main() -> None:
    ptwt = import_reference()
    bk = banks()
    arrays, man = {}, {"generated_by": "oracle/make_golden_banks.py", "torch": torch.__version__}
    for name, b in bk.items():
        arrays[f"{key_of(name)}_taps"] = np.array(b.filter_bank, dtype=np.float64)
    man["banks"] = {name: key_of(name) + "_taps" for name in bk}
    g = torch.Generator().manual_seed(20261016)

    cases = []

    def run(ndim, bank, mode, dtype, shape, level, axes):
        key = f"c{len(cases)}"
        dec, rec, axkw = transforms(ptwt, ndim)
        x = torch.randn(shape, generator=g, dtype=torch.float64).to(getattr(torch, dtype))
        kw = {} if axes is None else {axkw: axes}
        c = dec(x, bk[bank], mode=mode, level=level, **kw)
        y = rec(c, bk[bank], **kw)
        flat = flatten(c) + [y]
        arrays[f"{key}_x"] = x.numpy()
        arrays[f"{key}_o"] = torch.cat([t.reshape(-1) for t in flat]).numpy()
        cases.append(dict(key=key, ndim=ndim, bank=bank, mode=mode, dtype=dtype, shape=list(shape), level=level,
                          axes=list(axes) if isinstance(axes, tuple) else axes,
                          shapes=[list(t.shape) for t in flat]))

    for ndim in (1, 2, 3):
        for bank in BANKS:
            for mode in MODES:
                if ndim == 3 and mode in NEEDS_EXTENT:
                    # these volumes are large: one dtype per bank, both dtypes over the four banks
                    dtype = ("float64", "float32")[BANKS.index(bank) % 2]
                    run(ndim, bank, mode, dtype, shape_3d_long_pad(len(bk[bank])), 1, None)
                    continue
                run(ndim, bank, mode, "float64", SHAPES[ndim], None if ndim < 3 else 1, None)
                run(ndim, bank, mode, "float32", SHAPES_F32[ndim], LEVEL_F32[ndim], None)
        shape, axes, level = AXES_CASES[ndim]
        run(ndim, BANKS[(ndim - 1) % len(BANKS)], "reflect" if ndim < 3 else "zero", "float64", shape, level, axes)
    man["cases"] = cases

    packets = []
    for ndim, bank, mode, shape, maxlevel in PACKETS:
        key = f"p{len(packets)}"
        x = torch.randn(shape, generator=g, dtype=torch.float64)
        if ndim == 1:
            wp = ptwt.WaveletPacket(x, bk[bank], mode=mode, maxlevel=maxlevel)
            keys = wp.get_level(maxlevel, "natural")
        else:
            wp = ptwt.WaveletPacket2D(x, bk[bank], mode=mode, maxlevel=maxlevel)
            keys = wp.get_natural_order(maxlevel)
        wp.initialize(keys)
        every = sorted(k for k in wp.keys() if k != "")
        flat = [wp[k] for k in every] + [wp.reconstruct()[""]]
        arrays[f"{key}_x"] = x.numpy()
        arrays[f"{key}_o"] = torch.cat([t.reshape(-1) for t in flat]).numpy()
        packets.append(dict(key=key, ndim=ndim, bank=bank, mode=mode, shape=list(shape), maxlevel=maxlevel,
                            keys=every, shapes=[list(t.shape) for t in flat]))
    man["packets"] = packets

    grads = []
    for ndim, (bank, mode, shape, level) in GRAD_CASES.items():
        key = f"g{len(grads)}"
        dec, rec, _ = transforms(ptwt, ndim)
        x = torch.randn(shape, generator=g, dtype=torch.float64)
        taps = [torch.tensor(f, dtype=torch.float64, requires_grad=True) for f in bk[bank].filter_bank]
        xr = x.clone().requires_grad_(True)
        c = dec(xr, tuple(taps), mode=mode, level=level)
        y = rec(c, tuple(taps))
        flat = flatten(c)
        ws = [torch.randn(t.shape, generator=g, dtype=torch.float64) for t in flat]
        wy = torch.randn(y.shape, generator=g, dtype=torch.float64)
        loss = sum((w * t).sum() for w, t in zip(ws, flat)) + (wy * y).sum()
        loss.backward()
        arrays[f"{key}_x"] = x.numpy()
        arrays[f"{key}_w"] = torch.cat([w.reshape(-1) for w in ws + [wy]]).numpy()
        arrays[f"{key}_gx"] = xr.grad.numpy()
        arrays[f"{key}_gtaps"] = torch.stack([t.grad for t in taps]).numpy()
        grads.append(dict(key=key, ndim=ndim, bank=bank, mode=mode, shape=list(shape), level=level,
                          shapes=[list(t.shape) for t in flat + [y]], loss=float(loss.detach())))
    man["grads"] = grads

    np.savez_compressed(OUT / "bank_vectors.npz", **arrays)
    (OUT / "bank_vectors.json").write_text(json.dumps(man, indent=1) + "\n")
    print("wrote", OUT / "bank_vectors.npz", len(cases), "cases", len(packets), "packets", len(grads), "gradients",
          sum(v.nbytes for v in arrays.values()), "bytes raw", (OUT / "bank_vectors.npz").stat().st_size,
          "bytes compressed")


if __name__ == "__main__":
    main()
