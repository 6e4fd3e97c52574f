"""The oracle is only trusted once pinned: restatement == golden vectors produced by the unmodified reference (bit exact,
CPU fp32)."""
import pytest
import torch

from conftest import load_golden
from oracle import restatement as R


@pytest.mark.parametrize("name,lowres", [("unet_tiny_base.pt", False), ("unet_tiny_sr.pt", True)])
def test_restatement_matches_golden_unet(name, lowres):
    g = load_golden(name)
    inp = g["inputs"]
    kw = {k: v for k, v in inp.items() if k not in ("x", "time")}
    with torch.no_grad():
        assert torch.equal(R.unet_forward(g["state_dict"], g["cfg"], inp["x"], inp["time"], **kw), g["out_cond"])
        assert torch.equal(R.unet_forward(g["state_dict"], g["cfg"], inp["x"], inp["time"], cond_drop_prob=1., **kw),
                           g["out_null"])
        kw2 = dict(kw, text_mask=None)
        assert torch.equal(R.unet_forward(g["state_dict"], g["cfg"], inp["x"], inp["time"], **kw2), g["out_nomask"])
        cfg3 = R.cfg_combine(g["out_cond"], g["out_null"], 3.)
        assert torch.equal(cfg3, g["out_cfg3"])


@pytest.mark.parametrize("T", [25, 1000])
def test_restatement_matches_golden_step(T):
    g = load_golden("ddpm_step.pt")[T]
    tabs = R.ddpm_tables(T)
    for k, v in tabs.items():
        assert torch.equal(v, g["tables"][k]), k
    out = R.p_sample_step(tabs, g["x"], g["t"], g["eps"], g["noise"])
    assert torch.equal(out, g["out"])


def test_quantile_rank_is_fp32_arithmetic():
    """timestep-index / percentile-rank work is integer work: must be exact.  n = 3*1024^2 gives weight 0.25 because
    torch computes 0.9*(n-1) in fp32 (SURVEY.md 8a row 12)."""
    from minimagen_b200.Imagen import quantile_rank
    ranks = load_golden("ddpm_step.pt")["ranks"]
    assert ranks[3 * 1024 * 1024] == (2831154, 2831155, 0.25)
    for n, expect in ranks.items():
        assert quantile_rank(n, 0.9) == expect
        # and torch.quantile really behaves like sorted[lo] lerp sorted[hi] with that weight
    g = torch.Generator().manual_seed(0)
    x = torch.randn(4, 12288, generator=g).abs()
    lo, hi, w = quantile_rank(12288, 0.9)
    srt = x.sort(dim=-1).values
    assert torch.equal(torch.lerp(srt[:, lo], srt[:, hi], torch.tensor(w)), torch.quantile(x, 0.9, dim=-1))


def test_sample_loop_golden_matches_restatement():
    g = load_golden("sample_loop.pt")
    tabs = R.ddpm_tables(g["timesteps"])
    img = g["x_T"]
    with torch.no_grad():
        for i in range(3):
            t = torch.full((2,), g["timesteps"] - 1 - i)
            kw = dict(text_embeds=g["text_embeds"], text_mask=g["text_mask"])
            e = R.unet_forward(g["state_dict"], g["cfg"], img, t, **kw)
            n = R.unet_forward(g["state_dict"], g["cfg"], img, t, cond_drop_prob=1., **kw)
            img = R.p_sample_step(tabs, img, t, R.cfg_combine(e, n, g["cond_scale"]), g["noises"][i])
            assert torch.equal(img, g["traj"][i])


def test_restatement_matches_live_reference():
    """restatement == the unmodified reference on two further configurations (outputs recorded from the reference in
    tests/golden/reference_live.pt by oracle/make_golden.py live; the weights are this package's seeded initialisation)."""
    from minimagen_b200.Unet import Unet
    from oracle.make_golden import LIVE_CFGS, live_inputs
    g = load_golden("reference_live.pt")
    for (cfg, s, lowres), expect in zip(LIVE_CFGS, g["outputs"]):
        torch.manual_seed(0)
        sd = Unet(**cfg).state_dict()
        x, t, kw = live_inputs(cfg, s, lowres)
        with torch.no_grad():
            for cdp, e in zip((0., 1.), expect):
                assert torch.equal(R.unet_forward(sd, cfg, x, t, cond_drop_prob=cdp, **kw), e)
