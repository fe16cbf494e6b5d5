"""The fp16 mode (use_autocast=True) of whole networks.

Roformers (BS and Mel-Band, the small seeded golden models and one full-size released-geometry chunk) run against the operand-rounding
restatement (tests/fp16_operands.py: the unmodified oracle at float64 with both operands of every tensor-core contraction rounded to fp16).
Bounds, computed on the CPU in each test from the oracle itself (d16 = the restatement's max distance from the full-precision oracle):
  * fp16 net vs restatement: at most d16.  Per operator the kernels match the restatement to fp32 accumulation (test_autocast_ops_gpu.py),
    but end to end they cannot: rounding to fp16 is discontinuous, so the ~1e-7 fp32-vs-fp64 differences of the activations flip a few
    roundings in the first layer, each flip moves a GEMM output by a full fp16 step, and over a few layers the two computations decorrelate
    to about fp16 noise.  Measured on an H100: 0.66-0.75 d16 for the three Roformer models, 0.56 d16 for the small HTDemucs.  The bound says the kernels add nothing beyond fp16
    operand rounding.
  * fp16 net vs the fp32 golden: at most 1.5 d16 + 1e-5.
The small HTDemucs is held to the restatement the same way (its attention is SIMT-sized, its DConv layers run in the fused fp32 kernel).
HDemucs and VR (CascadedASPPNet and VR 5.1) have no restatement: VR folds BatchNorm into its weights before they are rounded, and the HDemucs
oracle writes its BLSTM projections as plain matrix products inside the recurrence, so neither can be rounded from outside the unmodified
oracle.  Their fp16 forwards are checked against the fp32 result with a signal-to-error floor.  For every net, test_every_tensor_core_launch_carries_the_mode
records the library calls of one forward and checks that each tensor-core launch carries the net's mode (so no class of launches is left in the
other mode), and every fp16 result is checked to differ from the default mode's."""
import os
from fractions import Fraction

import numpy as np
import pytest
import torch

import demucs_oracle as D
import mdx_oracle as M
import roformer_oracle as R
import vr_oracle as V
from fp16_operands import fp16_operands

pytestmark = pytest.mark.gpu

SMALL = dict(dim=32, depth=2, time_transformer_depth=1, freq_transformer_depth=2, freqs_per_bands=(2, 2, 4, 4, 8, 12, 16, 17), dim_head=8, heads=4, stft_n_fft=128,
             stft_hop_length=32, stft_win_length=128)
MSMALL = dict(dim=32, depth=2, time_transformer_depth=1, freq_transformer_depth=1, num_bands=12, dim_head=8, heads=4, mask_estimator_depth=2, stft_n_fft=128,
              stft_hop_length=32, stft_win_length=128)


def dev(x):
    return torch.as_tensor(np.ascontiguousarray(x)).cuda()


@pytest.fixture(scope="module")
def b200(lib_built):
    assert torch.cuda.is_available()
    from audio_separator.separator.b200 import _lib, demucs, roformer, vr

    return _lib, roformer, demucs, vr


def snr_db(got, ref):
    return 10 * np.log10(float(np.sum(ref.astype(np.float64) ** 2)) / max(float(np.sum((got.astype(np.float64) - ref) ** 2)), 1e-30))


def check_against_restatement(got, fwd, golden=None, **opts):
    """fwd(dtype) -> oracle output; see the module docstring for the two bounds"""
    with fp16_operands(**opts):
        r16 = fwd("float64")
    exact = fwd("float64")
    d16 = float(np.abs(r16 - exact).max())  # the oracle's own fp16-vs-full-precision distance
    assert d16 > 1e-6, "the fp16 restatement did not change the oracle: no tensor-core contraction in this model"
    err = float(np.abs(got - r16).max())
    assert err <= d16, (err, d16)
    if golden is not None:
        eg = float(np.abs(got - golden).max())
        assert eg <= 1.5 * d16 + 1e-5, (eg, d16)
    return err, d16


def test_bs_roformer_small_vs_restatement_and_golden(b200, golden_dir):
    _lib, rf, _, _ = b200
    gold = np.load(os.path.join(golden_dir, "roformer_small.npz"))
    ocfg = R.BSRoformerConfig(**dict(SMALL, dim_t=65, overlap=8))
    w = R.make_weights(ocfg, seed=3)
    mix = M.synth_music(int(gold["n_samples"]), seed=int(gold["mix_seed"]))[None, :, : ocfg.chunk_size]
    net = rf.BSRoformerNet(rf.BSRoformerConfig(**SMALL), w, math=_lib.MATH_FP16)
    got = net.forward(dev(mix)).cpu().numpy()
    _, d16 = check_against_restatement(got, lambda dt: R.forward(w, ocfg, mix, dtype=dt), gold["forward_ref"])
    got32 = rf.BSRoformerNet(rf.BSRoformerConfig(**SMALL), w).forward(dev(mix)).cpu().numpy()
    assert np.abs(got32 - gold["forward_ref"]).max() <= 1e-4  # the default mode of a second net is untouched
    assert np.abs(got - got32).max() > 0.1 * d16  # the fp16 mode is in effect


def test_mel_roformer_small_vs_restatement_and_golden(b200, golden_dir):
    _lib, rf, _, _ = b200
    gold = np.load(os.path.join(golden_dir, "roformer_small.npz"))
    ocfg = R.MelBandRoformerConfig(**dict(MSMALL, dim_t=65))
    w = R.make_mel_weights(ocfg, seed=6)
    mix = M.synth_music(int(gold["n_samples"]), seed=int(gold["mix_seed"]))[None, :, : ocfg.chunk_size]
    got = rf.BSRoformerNet(rf.MelBandRoformerConfig(**MSMALL), w, math=_lib.MATH_FP16).forward(dev(mix)).cpu().numpy()
    _, d16 = check_against_restatement(got, lambda dt: R.forward_mel(w, ocfg, mix, dtype=dt), gold["mel_forward_ref"])
    got32 = rf.BSRoformerNet(rf.MelBandRoformerConfig(**MSMALL), w).forward(dev(mix)).cpu().numpy()
    assert np.abs(got - got32).max() > 0.1 * d16  # the fp16 mode is in effect


def test_bs_roformer_full_size_chunk_vs_restatement(b200):
    """The released geometry (dim 512, depth 12, 8 heads x 64 -> the fused attention kernel in fp16, 62 bands, 801 frames)."""
    _lib, rf, _, _ = b200
    kw = dict(stft_hop_length=441)
    ocfg = R.BSRoformerConfig(**kw)
    w = R.make_weights(ocfg, seed=8)
    mix = M.synth_music(ocfg.chunk_size, seed=9)[None]
    mix = (mix / np.abs(mix).max() * 0.9).astype(np.float32)
    got = rf.BSRoformerNet(rf.BSRoformerConfig(**kw), w, math=_lib.MATH_FP16).forward(dev(mix)).cpu().numpy()
    err, d16 = check_against_restatement(got, lambda dt: R.forward(w, ocfg, mix, dtype=dt))
    got32 = rf.BSRoformerNet(rf.BSRoformerConfig(**kw), w).forward(dev(mix)).cpu().numpy()
    assert np.abs(got - got32).max() > 0.1 * d16  # the fp16 mode is in effect
    print(f"full-size BS-Roformer chunk: |fp16 net - restatement| {err:.3e}, |restatement - fp64| {d16:.3e}")


def test_htdemucs_small_vs_restatement_and_golden(b200, golden_dir):
    """HTDemucs (head dimension 8: the attention products are SIMT-sized and stay fp32; the fused DConv layers stay fp32): every convolution,
    transposed convolution and linear that the library sends to the tensor cores is rounded in the restatement."""
    _lib, _, dm, _ = b200
    z = np.load(os.path.join(golden_dir, "demucs_small.npz"))
    kw = dict(channels=8, bottom_channels=32, t_layers=3, t_heads=4, segment=Fraction(1, 2))
    ocfg = D.HTConfig(**kw)
    w = D.make_weights(ocfg, seed=int(z["weights_seed"]))
    mix = M.synth_music(3 * ocfg.seg_len, seed=int(z["mix_seed"]))[None, :, : ocfg.seg_len]
    y16 = dm.HTDemucsNet(dm.HTDemucsConfig(**kw), w, math=_lib.MATH_FP16).forward(dev(mix)).cpu().numpy()
    y32 = dm.HTDemucsNet(dm.HTDemucsConfig(**kw), w).forward(dev(mix)).cpu().numpy()
    assert np.abs(y32 - z["forward_ref"]).max() <= 1e-4
    err, d16 = check_against_restatement(y16, lambda dt: D.forward(w, ocfg, mix, dtype=dt), z["forward_ref"], dconv_fused_hid=dm._DCONV_FUSED_HID)
    assert np.abs(y16 - y32).max() > 0.1 * d16  # the fp16 mode is in effect
    print(f"small HTDemucs: |fp16 net - restatement| {err:.3e}, |restatement - fp64| {d16:.3e}")


def test_hdemucs_small_fp16(b200, golden_dir):
    import hdemucs_oracle as H
    from audio_separator.separator.b200 import hdemucs as hd

    _lib = b200[0]
    z = np.load(os.path.join(golden_dir, "hdemucs_small.npz"))
    kw = dict(channels=8, nfft=256, depth=4, norm_starts=2, dconv_lstm=2, dconv_attn=2, segment=0.5)
    w = H.make_weights(H.HDConfig(**kw), seed=int(z["weights_seed"]))
    mix = M.synth_music(3 * H.HDConfig(**kw).seg_len, seed=int(z["mix_seed"]))[None, :, : H.HDConfig(**kw).seg_len]
    y16 = hd.HDemucsNet(hd.HDemucsConfig(**kw), w, math=_lib.MATH_FP16).forward(dev(mix)).cpu().numpy()
    y32 = hd.HDemucsNet(hd.HDemucsConfig(**kw), w).forward(dev(mix)).cpu().numpy()
    assert np.isfinite(y16).all() and np.abs(y16 - y32).max() > 1e-5
    s = snr_db(y16, y32)
    print(f"small HDemucs: fp16 vs bf16x3 {s:.1f} dB")
    assert s >= 50.0, s  # measured on an H100: 64.8 dB


@pytest.mark.parametrize("arch,bins", [(31191, 128), (129605, 128), ("5.1", 128)])
def test_vr_fp16(b200, golden_dir, arch, bins):
    _lib, _, _, vr = b200
    gold = np.load(os.path.join(golden_dir, "vr_small.npz"))
    if arch == "5.1":
        w = V.make_weights_51(256, 8, 16, seed=3)
        make = lambda math: vr.VRNet51(256, 8, 16, w, math=math)  # noqa: E731
        x, ref = dev(gold["mask51_in"]), gold["mask51_ref"]
    else:
        w = V.make_weights(arch, seed=arch % 97)
        make = lambda math: vr.VRNet(arch, bins * 2, w, math=math)  # noqa: E731
        x, ref = dev(gold[f"mask_in_{arch}"]), gold[f"mask_ref_{arch}"]
    m16 = make(_lib.MATH_FP16).predict_mask(x).cpu().numpy()
    m32 = make(_lib.MATH_BF16X3).predict_mask(x).cpu().numpy()
    assert np.abs(m32 - ref).max() <= 1e-4
    assert np.isfinite(m16).all() and np.abs(m16 - m32).max() > 1e-6
    s = snr_db(m16, ref)
    print(f"VR {arch}: fp16 vs golden {s:.1f} dB")
    assert s >= 50.0, s  # measured on an H100: 56.4 / 72.0 / 75.2 dB


# ------------------------------------------------------------------------------------------------ every launch carries the net's mode
_MATH_ENTRIES = {"b200sep_gemm_f32_math": 20, "b200sep_conv2d_f32_math": 29, "b200sep_attention_f32_math": 20, "b200sep_attention_work_floats_math": 4,
                 "b200sep_tc_packed_floats_math": 2, "b200sep_tc_pack_linear_weights_math": 5, "b200sep_tc_pack_conv_weights_math": 5}  # name: index of `math`
_PLAIN_ENTRIES = ("b200sep_gemm_f32", "b200sep_conv2d_f32", "b200sep_attention_f32", "b200sep_attention_work_floats", "b200sep_tc_packed_floats",
                  "b200sep_tc_pack_linear_weights", "b200sep_tc_pack_conv_weights")


class LaunchLog:
    """Wraps the tensor-core entry points of the loaded library: records the math argument of every *_math call and counts calls of the entries
    without the suffix (which always mean BF16X3)."""

    def __init__(self, lib):
        self.lib, self.modes, self.plain, self.saved = lib, [], [], {}

    def __enter__(self):
        for name in list(_MATH_ENTRIES) + list(_PLAIN_ENTRIES):
            fn = getattr(self.lib, name)
            self.saved[name] = fn

            def wrap(*a, _fn=fn, _name=name):
                if _name in _MATH_ENTRIES:
                    self.modes.append((_name, a[_MATH_ENTRIES[_name]]))
                else:
                    self.plain.append(_name)
                return _fn(*a)

            setattr(self.lib, name, wrap)
        return self

    def __exit__(self, *exc):
        for name, fn in self.saved.items():
            setattr(self.lib, name, fn)


@pytest.mark.parametrize("net", ["bs_roformer", "htdemucs", "hdemucs", "vr", "vr51"])
def test_every_tensor_core_launch_carries_the_mode(b200, net):
    """A net built with math=m issues every gemm / conv / attention launch (and every packing) with m, and never the suffix-less BF16X3 entries."""
    _lib, rf, dm, vr = b200
    g = np.random.default_rng(0)
    if net == "bs_roformer":
        ocfg = R.BSRoformerConfig(**dict(SMALL, dim_t=65))
        w = R.make_weights(ocfg, seed=3)
        build = lambda m: rf.BSRoformerNet(rf.BSRoformerConfig(**SMALL), w, math=m)  # noqa: E731
        x = dev(M.synth_music(ocfg.chunk_size, seed=1)[None])
    elif net == "htdemucs":
        kw = dict(channels=8, bottom_channels=32, t_layers=3, t_heads=4, segment=Fraction(1, 2))
        w = D.make_weights(D.HTConfig(**kw), seed=2)
        build = lambda m: dm.HTDemucsNet(dm.HTDemucsConfig(**kw), w, math=m)  # noqa: E731
        x = dev(M.synth_music(D.HTConfig(**kw).seg_len, seed=1)[None])
    elif net == "hdemucs":
        import hdemucs_oracle as H
        from audio_separator.separator.b200 import hdemucs as hd

        kw = dict(channels=8, nfft=256, depth=4, norm_starts=2, dconv_lstm=2, dconv_attn=2, segment=0.5)
        w = H.make_weights(H.HDConfig(**kw), seed=2)
        build = lambda m: hd.HDemucsNet(hd.HDemucsConfig(**kw), w, math=m)  # noqa: E731
        x = dev(M.synth_music(H.HDConfig(**kw).seg_len, seed=1)[None])
    elif net == "vr":
        w = V.make_weights(31191, seed=5)
        build = lambda m: vr.VRNet(31191, 256, w, math=m)  # noqa: E731
        x = dev(np.abs(g.standard_normal((2, 2, 129, 272))).astype(np.float32))
    else:
        w = V.make_weights_51(256, 8, 16, seed=3)
        build = lambda m: vr.VRNet51(256, 8, 16, w, math=m)  # noqa: E731
        x = dev(np.abs(g.standard_normal((2, 2, 129, 160))).astype(np.float32))
    for m in (_lib.MATH_FP16, _lib.MATH_BF16X3):
        model = build(m)
        with LaunchLog(_lib.lib) as log:
            (model.predict_mask if net.startswith("vr") else model.forward)(x)
            torch.cuda.synchronize()
        assert log.plain == [], log.plain
        assert len(log.modes) >= 5 and {mode for _, mode in log.modes} == {m}, (m, sorted(set(log.modes)))
