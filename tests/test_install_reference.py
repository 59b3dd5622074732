"""install() / uninstall() on a package with the reference's module layout (tests/stand_in_ptwt.py): rebinding in ptwt
and in the modules that captured the names by value, and the numbers and gradients of the unmodified reference
(stored by oracle/make_golden_api.py) reproduced by the new kernels."""
from __future__ import annotations

import pytest
import torch

import pytorch_wavelet_toolbox_b200 as wt
from conftest import flatten_coeffs
from stand_in_ptwt import stand_in_ptwt

pytestmark = pytest.mark.gpu


@pytest.fixture
def ptwt():
    with stand_in_ptwt() as mod:
        yield mod


def test_install_rebinds_and_uninstall_restores(ptwt, reference_api):
    packets, sep = ptwt.packets, ptwt.separable_conv_transform
    manifest, arrays = reference_api
    ref_wavedec, ref_packets_wavedec, ref_sep_wavedec = ptwt.wavedec, packets.wavedec, sep.wavedec
    replaced = wt.install()
    assert "ptwt.wavedec" in replaced and "ptwt.packets.wavedec" in replaced
    assert ptwt.wavedec is wt.wavedec and packets.wavedec is wt.wavedec and sep.wavedec is wt.wavedec
    assert ptwt.conv_transform_2.wavedec2 is wt.wavedec2 and ptwt.matmul_transform.MatrixWavedec is wt.MatrixWavedec
    assert ptwt.WaveletPacket is wt.WaveletPacket and packets.WaveletPacket2D is wt.WaveletPacket2D
    x = torch.from_numpy(arrays["install_x"]).cuda()
    got = ptwt.wavedec2(x, "db2", level=2)                      # the reference's name, our kernels
    wt.uninstall()
    assert ptwt.wavedec is ref_wavedec and packets.wavedec is ref_packets_wavedec and sep.wavedec is ref_sep_wavedec
    want = [torch.from_numpy(arrays[f"install_o{j}"]) for j in range(manifest["install_n_out"])]
    scale = max(float(t.abs().max()) for t in want)
    flat = flatten_coeffs(got)
    assert len(flat) == len(want)
    for a, b in zip(flat, want):
        assert a.is_cuda and float((a.cpu() - b).abs().max()) <= 1e-5 * scale


def test_learnable_filters_receive_the_reference_gradients(reference_api):
    """Filter taps as nn.Parameters (the reference's learnable ProductFilter, wavelets_learnable.py:167-199, trained
    through wavedec / waverec as in examples/network_compression/wavelet_linear.py:118,150): the loss, the data and
    the four filters receive the gradients the reference computed."""
    manifest, arrays = reference_api
    spec = manifest["learnable"]
    fb = wt.WaveletTensorTuple.from_wavelet(wt._wavelets.as_wavelet(spec["wavelet"]), torch.float64)
    wav = wt.WaveletTensorTuple(*[torch.nn.Parameter(t.clone()) for t in fb])
    x = torch.from_numpy(arrays["learn_x"])
    w = torch.from_numpy(arrays["learn_w"])
    n = x.shape[-1]
    xo = x.clone().cuda().requires_grad_(True)
    c = wt.wavedec(xo, wav, level=spec["level"], mode=spec["mode"])
    rec = wt.waverec(c, wav)[..., :n]
    loss = sum((t * t).sum() for t in c) + (rec * w.cuda()).sum()
    loss.backward()
    assert abs(float(loss) - spec["loss"]) <= 1e-10 * abs(spec["loss"])
    want = torch.from_numpy(arrays["learn_grad_x"])
    assert float((xo.grad.cpu() - want).abs().max()) <= 1e-10 * float(want.abs().max())
    for name in ("dec_lo", "dec_hi", "rec_lo", "rec_hi"):
        a, b = getattr(wav, name).grad, torch.from_numpy(arrays[f"learn_grad_{name}"])
        assert a is not None, name
        assert float((a.cpu() - b).abs().max()) <= 1e-9 * float(b.abs().max()), name
