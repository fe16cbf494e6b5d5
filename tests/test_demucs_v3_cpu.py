"""CPU checks of the time-domain Demucs v3 path: the oracle against the reference-generated golden, the product's layer plan / state-key mapping /
valid_length against the oracle and the reference's values, the package loader's dispatch, and the julius filter tables."""
import math
import os
import sys
import types

import numpy as np
import pytest
import torch

import demucs_v3_oracle as V
import hdemucs_oracle as H
import mdx_oracle as M

SMALL = dict(channels=8, depth=4, norm_starts=2, dconv_lstm=2, dconv_attn=2, dconv_mode=3, segment=0.1)
SMALL_B = dict(channels=8, depth=3, dconv_mode=1, context=0, segment=0.15)
HD_SMALL = dict(channels=8, nfft=256, depth=4, norm_starts=2, dconv_lstm=2, dconv_attn=2, segment=0.5)


@pytest.fixture(scope="module")
def gold(golden_dir):
    return np.load(os.path.join(golden_dir, "demucs_v3_small.npz"))


def test_oracle_matches_reference_golden(gold):
    z = gold
    cfg = V.V3Config(**SMALL)
    w = V.make_weights(cfg, seed=int(z["weights_seed"][0]))
    mix = M.synth_music(3 * int(z["n_apply"]), seed=int(z["mix_seed"]))
    n, nl = int(z["fwd_len"]), int(z["long_len"])
    assert np.abs(V.forward(w, cfg, mix[None, :, :n]) - z["forward_b2_ref"][:1]).max() <= 5e-5  # one chunk = entry 0 of the batch-2 golden
    assert np.abs(V.forward(w, cfg, mix[None, :, :nl]) - z["forward_long_ref"]).max() <= 5e-5
    cfg_b, hcfg = V.V3Config(**SMALL_B), H.HDConfig(**HD_SMALL)
    w_b, hw = V.make_weights(cfg_b, seed=int(z["weights_seed"][1])), H.make_weights(hcfg, seed=int(z["weights_seed"][2]))
    m2 = torch.from_numpy(mix[:, : int(z["n_apply"])])
    mn = ((m2 - m2.mean(0).mean()) / m2.mean(0).std()).numpy()[None]
    members = [(lambda c: V.forward(w, cfg, c), cfg), (lambda c: V.forward(w_b, cfg_b, c), cfg_b), (lambda c: H.forward(hw, hcfg, c), hcfg)]
    got = V.apply_bag(members, z["bag_weights"].tolist(), mn, z["bag_nosplit_offsets"].tolist(), split=False)
    assert np.abs(got - z["bag_nosplit_ref"]).max() <= 5e-5 * np.abs(z["bag_nosplit_ref"]).max()


def test_layer_plan_state_keys_and_valid_length(lib_built, gold):
    from audio_separator.separator.b200 import demucs_v3 as dv

    cfg = dv.DemucsConfig(channels=48)
    assert [cfg.valid_length(int(n)) for n in gold["valid_in"]] == gold["valid_ref"].tolist()  # Demucs.valid_length of the reference
    assert all(cfg.valid_length(cfg.valid_length(n)) == cfg.valid_length(n) and cfg.valid_length(n) % 2 == 0 for n in range(1, 30000, 37))
    plan = dv.layer_plan(cfg)
    assert [(P["enc"]["chin"], P["enc"]["chout"], P["dec"]["chin"], P["dec"]["chout"]) for P in plan] == [
        (2, 48, 48, 8), (48, 96, 96, 48), (96, 192, 192, 96), (192, 384, 384, 192), (384, 768, 768, 384), (768, 1536, 1536, 768)]
    assert [(P["enc"]["norm"], P["enc"]["lstm"], P["dec"]["norm_tr"], P["dec"]["last"]) for P in plan] == [(False, False, False, True)] + [(False, False, False, False)] * 3 + [
        (True, True, True, False)] * 2
    assert all(P["enc"]["pad"] == 0 and P["enc"]["context"] == 0 and P["dec"]["context"] == 1 for P in plan)
    # every parameter of the reference layout (the oracle's param_shapes are asserted equal to the reference state_dict when the golden is made) maps onto a
    # name the layers read, and the structure check accepts exactly that set
    for kw in (dict(channels=48), SMALL, SMALL_B, dict(SMALL, norm_starts=0), dict(SMALL, dconv_mode=2)):
        c = dv.DemucsConfig(**kw)
        st = dict(V.make_weights(V.V3Config(**kw), seed=0))
        named = dv.layer_names(c, st)
        assert len(named) == len(st) and all(k.split(".")[2] in ("conv", "norm1", "dconv", "rewrite", "norm2", "conv_tr") for k in named)
        net = types.SimpleNamespace(cfg=c, encs=[(f"encoder.{i}", P["enc"]) for i, P in enumerate(dv.layer_plan(c))],
                                    decs=[(f"decoder.{j}", P["dec"]) for j, P in enumerate(dv.layer_plan(c)[::-1])])
        dv.DemucsNet._check_structure(net, named)
        bad = dict(named)
        bad.pop(next(k for k in named if ".norm" in k or ".rewrite." in k))
        with pytest.raises(ValueError):
            dv.DemucsNet._check_structure(net, bad)
    # the previous generation's `.2.` rewrite keys load like Demucs.load_state_dict renames them (demucs.py:444-453)
    c = dv.DemucsConfig(**dict(SMALL_B, dconv_mode=0))
    st = V.make_weights(V.V3Config(**dict(SMALL_B, dconv_mode=0)), seed=0)
    old = {k.replace("encoder.1.3.", "encoder.1.2."): v for k, v in st.items()}
    assert dv.layer_names(c, old).keys() == dv.layer_names(c, st).keys()
    with pytest.raises(ValueError):
        dv.layer_names(c, dict(st, **{"lstm.lstm.weight_ih_l0": np.zeros(1)}))


def _package(path, module, kwargs, state, name="Demucs"):
    parts = module.split(".")
    mods = {".".join(parts[: i + 1]): types.ModuleType(".".join(parts[: i + 1])) for i in range(len(parts))}
    K = type(name, (), {"__module__": module})
    setattr(mods[module], name, K)
    saved = {m: sys.modules.get(m) for m in mods}
    sys.modules.update(mods)
    try:
        torch.save({"klass": K, "args": (), "kwargs": kwargs, "state": state}, path)
    finally:
        for m, v in saved.items():
            if v is None:
                del sys.modules[m]
            else:
                sys.modules[m] = v


def test_loader_dispatch(lib_built, tmp_path):
    from audio_separator.separator.b200 import demucs_loader as L
    from audio_separator.separator.b200.demucs_v3 import DemucsConfig

    cfg = V.V3Config(**SMALL)
    state = {k: torch.from_numpy(v).half() for k, v in V.make_weights(cfg, seed=3).items()}
    kw = dict(cfg.kwargs(), rescale=0.1, dconv_init=1e-4, lstm_layers=0, glu=True, gelu=True, rewrite=True, normalize=True, resample=True)
    _package(str(tmp_path / "v3.th"), "demucs.demucs", kw, state)
    (models, wts, seg) = L.load_demucs(str(tmp_path / "v3.th"))
    c, st = models[0]
    assert isinstance(c, DemucsConfig) and (c.channels, c.depth, c.norm_starts, c.dconv_mode, c.segment, c.sources) == (8, 4, 2, 3, 0.1, ("drums", "bass", "other", "vocals"))
    assert set(st) == set(state) and all(v.dtype == np.float32 for v in st.values())
    _package(str(tmp_path / "defaults.th"), "demucs.demucs", {"sources": ["a", "b"]}, state)
    c2 = L.config_from_package(L.load_package(str(tmp_path / "defaults.th")))
    assert (c2.channels, c2.segment, c2.growth, c2.depth) == (64, 40.0, 2.0, 6)  # constructor defaults (demucs.py:236-272)
    for module in ("demucs.model", "demucs.model_v2", "demucs.tasnet", "demucs_fake_pkg.htdemucs"):  # v1 / v2 packages share the class name
        _package(str(tmp_path / "v2.th"), module, kw, state)
        with pytest.raises(NotImplementedError):
            L.config_from_package(L.load_package(str(tmp_path / "v2.th")))
    for bad in (dict(lstm_layers=2), dict(glu=False), dict(gelu=False), dict(rewrite=False), dict(normalize=False), dict(resample=False), dict(kernel_size=6)):
        _package(str(tmp_path / "bad.th"), "demucs.demucs", dict(kw, **bad), state)
        with pytest.raises(NotImplementedError):
            L.config_from_package(L.load_package(str(tmp_path / "bad.th")))


def test_julius_taps_closed_form(lib_built):
    from audio_separator.separator.b200.demucs_v3 import julius_taps

    for old, new, width, n in ((1, 2, 26, 53), (2, 1, 51, 104)):
        k, w = julius_taps(old, new)
        assert w == width and k.shape == (new, n)
        assert np.abs(k - V.julius_taps(old, new)[0]).max() == 0.0
        sr = min(old, new) * 0.945
        for i in range(new):
            for j in range(n):
                t = min(max((-i / new + (j - width) / old) * sr, -24.0), 24.0) * math.pi
                v = (1.0 if t == 0 else math.sin(t) / t) * math.cos(t / 48) ** 2
                assert abs(k[i, j] * sum((1.0 if tt == 0 else math.sin(tt) / tt) * math.cos(tt / 48) ** 2 for tt in
                                         (min(max((-i / new + (jj - width) / old) * sr, -24.0), 24.0) * math.pi for jj in range(n))) - v) <= 1e-12
            assert abs(k[i].sum() - 1.0) <= 1e-12
    k, _ = julius_taps(1, 2)
    assert np.allclose(k[0], k[0][::-1]) and np.allclose(k[1][1:], k[1][1:][::-1])  # phase 0 centred on a sample, phase 1 half-way to the next


def test_resample_round_trip_band_limited():
    g = torch.Generator().manual_seed(0)
    n = 20000
    t = torch.arange(n, dtype=torch.float64)
    f = torch.rand(24, generator=g, dtype=torch.float64) * 0.4  # cycles per sample, below the 0.945 / 2 roll-off of the /2 filter
    x = sum(torch.cos(2 * math.pi * fi * t + 6.0 * torch.rand(1, generator=g, dtype=torch.float64)) for fi in f)[None, None]
    y = V.resample_frac(V.resample_frac(x, 1, 2), 2, 1)
    assert y.shape == x.shape
    inner = slice(200, n - 200)
    err = (y - x)[..., inner].abs().max() / x.abs().max()
    assert err <= 2e-3, float(err)
