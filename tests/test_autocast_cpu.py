"""CPU: which architectures use_autocast switches to the fp16 tensor-core mode, and the operand-rounding restatement the GPU tests use."""
import numpy as np
import torch
import torch.nn.functional as F

import roformer_oracle as R
from fp16_operands import fp16_operands, tc_gemm_usable


def test_architecture_to_math_mode(lib_built):
    from audio_separator.separator.b200._lib import MATH_BF16X3, MATH_FP16
    from audio_separator.separator.common_separator import CommonSeparator, tensor_core_math

    for arch in ("Demucs", "VR", "Roformer"):
        assert tensor_core_math(arch, True) == MATH_FP16
        assert tensor_core_math(arch, False) == MATH_BF16X3
        assert tensor_core_math(arch, None) == MATH_BF16X3  # a common config without the key
    for arch in ("MDX", "MDX23C"):  # ONNX Runtime in the reference (autocast has no effect) / pair-format kernels without an fp16 mode
        assert tensor_core_math(arch, True) == MATH_BF16X3
    assert "use_autocast" in CommonSeparator._CONFIG_KEYS


def test_restatement_rounds_only_tensor_core_contractions():
    g = torch.Generator().manual_seed(0)
    big_x, big_w = torch.randn((200, 64), generator=g, dtype=torch.float64), torch.randn((96, 64), generator=g, dtype=torch.float64)
    small_w = torch.randn((8, 64), generator=g, dtype=torch.float64)  # N < 32: the SIMT kernel, fp32 in every mode
    assert tc_gemm_usable(200, 96, 64) and not tc_gemm_usable(200, 8, 64)
    linear0 = F.linear
    with fp16_operands():
        y = F.linear(big_x, big_w, torch.ones(96, dtype=torch.float64))
        ys = F.linear(big_x, small_w)
    assert F.linear is linear0  # restored
    ref = big_x.half().double() @ big_w.half().double().t() + 1.0
    assert torch.equal(y, ref)
    assert torch.equal(ys, big_x @ small_w.t())
    assert torch.equal(torch.tensor([70000.0]).half().double(), torch.tensor([float("inf")], dtype=torch.float64))  # overflow: +-inf, not clamped


def test_restated_roformer_stays_close_to_the_oracle():
    """The fp16 restatement of a small BS-Roformer differs from the float64 oracle by fp16-sized amounts (it does round something)."""
    kw = dict(dim=64, depth=1, time_transformer_depth=1, freq_transformer_depth=1, freqs_per_bands=(2, 2, 4, 4, 8, 12, 16, 17), dim_head=64, heads=2,
              stft_n_fft=128, stft_hop_length=32, stft_win_length=128)
    ocfg = R.BSRoformerConfig(**dict(kw, dim_t=65))
    w = R.make_weights(ocfg, seed=1)
    import mdx_oracle as M

    mix = M.synth_music(ocfg.chunk_size, seed=2)[None]
    exact = R.forward(w, ocfg, mix, dtype="float64")
    with fp16_operands():
        r16 = R.forward(w, ocfg, mix, dtype="float64")
    d = np.abs(r16 - exact).max()
    assert 1e-6 < d < 1e-2 * max(1.0, np.abs(exact).max()), d
