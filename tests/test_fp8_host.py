"""FP8 mode, host side: its CPU emulation (tests/fp8_emulation.py, on top of the unchanged oracle) and the configuration check that runs
before any device work.

Emulated FP8 against the reference goldens (fp32 reference, synthetic weights), measured on the CPU oracle:
    dit_tiny72  max 0.236  mean 0.038      dit_tiny64  max 0.162  mean 0.029
    dit_L_c1    max 0.206  mean 0.043      dit_XL      max 0.218  mean 0.034      (outputs of mean |x| 0.75 .. 0.95)
The bound FP8_TOL = (0.35, 0.06) keeps about 1.5x over the largest of them.  It is the accuracy the FP8 mode trades for speed: every QKV
and GEGLU operand carries e4m3's 3-bit mantissa (2^-4 relative rounding) into the residual stream of every block."""
import pytest
import torch

from oracle import ezaudio_oracle as O
from tests import fp8_emulation as E
from tests import helpers

FP8_TOL = (0.35, 0.06)


def _all_finite_e4m3():
    codes = torch.arange(256, dtype=torch.int32).to(torch.uint8).view(torch.float8_e4m3fn).float()
    return codes[torch.isfinite(codes)]


def test_fp8_rows_round_trips_e4m3():
    v = _all_finite_e4m3()
    assert float(v.abs().max()) == 448.0 and v.numel() == 254
    for scale in (1.0, 2.0 ** -5, 2.0 ** 7):   # power-of-two scales: every e4m3 value comes back exactly
        x = (v * scale)[None]
        assert torch.equal(E.fp8_rows(x), x), scale
    # arbitrary rows: round to nearest even with saturation, exactly as torch's float8_e4m3fn cast of x * 448 / amax
    g = torch.Generator().manual_seed(0)
    x = torch.randn(64, 1152, generator=g) * torch.rand(64, 1, generator=g) * 10
    amax = x.abs().amax(-1, keepdim=True)
    want = (x * (448.0 / amax)).to(torch.float8_e4m3fn).float() * (amax / 448.0)
    assert torch.equal(E.fp8_rows(x), want)
    assert float((E.fp8_rows(x) - x).abs().div(amax).max()) <= 2.0 ** -4 * 448 / 448   # half a step of the top binade, relative to amax
    z = torch.zeros(2, 16)
    assert torch.equal(E.fp8_rows(z), z)                # amax = 0: scale 0, no division by zero
    assert E.fp8_rows(x.double()).dtype == torch.float64


def test_fp8_emulation_touches_only_the_two_projections(monkeypatch):
    cfg, sd, inp, _ = helpers.dit_case_inputs("dit_tiny72")
    seen = []
    lin = O.F.linear
    monkeypatch.setattr(O.F, "linear", lambda x, w, b=None: seen.append(w) or lin(x, w, b))
    with torch.no_grad():
        E.maskdit_forward(sd, cfg, inp["x"], inp["t"], inp["ctx"], inp["mask"])
    exact = {id(v) for v in sd.values()}
    swapped = [w for w in seen if id(w) not in exact]   # weights the emulation replaced by their e4m3 version
    n_blocks = cfg["depth"] + 1
    assert len(swapped) == 4 * n_blocks and all(torch.equal(E.fp8_rows(w), w) for w in swapped)
    assert O.attention is not None and O.attention.__name__ == "attention"   # the oracle is restored afterwards


@pytest.mark.parametrize("name", ["dit_tiny72", "dit_tiny64", "dit_L_c1", pytest.param("dit_XL", marks=pytest.mark.slow)])
def test_fp8_emulation_against_reference_golden(name):
    cfg, sd, inp, g = helpers.dit_case_inputs(name)
    with torch.no_grad():
        out, _ = E.maskdit_forward(sd, cfg, inp["x"], inp["t"], inp["ctx"], inp["mask"], inp["gt"], inp["gt_mask"])
    err = (helpers.golden_view(g, out) - torch.from_numpy(g["out"])).abs()
    print(f"[fp8 emulation] {name}: max-abs {float(err.max()):.3e} mean-abs {float(err.mean()):.3e}")
    assert float(err.max()) < FP8_TOL[0] and float(err.mean()) < FP8_TOL[1]
    assert float(err.mean()) > 1e-3   # the emulation is on: fp32 alone sits at ~1e-5


@pytest.mark.parametrize("head_dim,heads", [(96, 2), (72, 3)])   # no packed-QKV kernel: head dim not 64 / 72, odd head count
def test_fp8_rejects_unsupported_configs_before_device_work(head_dim, heads, monkeypatch):
    from ezaudio_b200 import _lib, synth
    from ezaudio_b200.dit import MaskDiT

    def no_device(*a, **k):
        raise AssertionError("device work before the configuration check")
    monkeypatch.setattr(_lib, "lib", no_device)
    cfg = synth.tiny_model(head_dim, heads=heads)
    with pytest.raises(ValueError, match="fp8"):
        MaskDiT(precision="fp8", max_batch=1, max_len=8, max_ctx_len=4, max_timesteps=2, **cfg)
