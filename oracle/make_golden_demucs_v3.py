"""Pin oracle/demucs_v3_oracle.py against the UNMODIFIED reference Demucs (+ apply_model on a BagOfModels) and write tests/golden/demucs_v3_small.npz.

julius is not installed: ref_shim registers an empty stand-in module, and this script gives it the oracle's resample_frac before the reference
runs, so the resampling step is the same restatement on both sides ("parity unpinned"); everything else is the reference's own code."""
import os
import random
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import demucs_v3_oracle as V  # noqa: E402
import hdemucs_oracle as H  # noqa: E402
import mdx_oracle as M  # noqa: E402
import ref_shim  # noqa: E402
from make_golden import check  # noqa: E402
from make_golden_hdemucs import SMALL as HD_SMALL, ref_model as hd_ref_model  # noqa: E402

GOLD = os.path.join(os.path.dirname(HERE), "tests", "golden")
# depth 4: DConv in encoder and decoder, GroupNorm / BLSTM / LocalState from index 2 on (the layer kinds of the released depth-6 models, whose
# norm_starts = dconv_lstm = dconv_attn = 4); the second member: depth 3, encoder-only DConv, no GroupNorm, another segment.  Short segments
# give the short bag input several overlapping chunks per member, and the ragged length is the shortest that frames the index-2 BLSTM (204 steps),
# so the golden stays small
SMALL = dict(channels=8, depth=4, norm_starts=2, dconv_lstm=2, dconv_attn=2, dconv_mode=3, segment=0.1)
SMALL_B = dict(channels=8, depth=3, dconv_mode=1, context=0, segment=0.15)
BAG_WEIGHTS = [[1.0, 0.5, 1.0, 0.0], [0.5, 1.0, 0.0, 1.0], [1.0, 1.0, 1.0, 1.0]]
FWD_LEN, LONG_LEN, N_APPLY = 2000, 6451, 3000


def ref_model(cfg, w):
    dm = ref_shim.ref_module("audio_separator.separator.uvr_lib_v5.demucs.demucs")
    m = dm.Demucs(**cfg.kwargs()).eval()
    sd = m.state_dict()
    shapes = dict(V.param_shapes(cfg))
    assert list(sd) == list(shapes), [(a, b) for a, b in zip(sd, shapes) if a != b][:5] + [len(sd), len(shapes)]
    for n, v in sd.items():
        assert tuple(v.shape) == shapes[n], (n, v.shape, shapes[n])
    m.load_state_dict({k: torch.from_numpy(v) for k, v in w.items()})
    return m


def main():
    ref_shim.install()
    sys.modules["julius"].resample_frac = V.resample_frac
    cfg, cfg_b, hcfg = V.V3Config(**SMALL), V.V3Config(**SMALL_B), H.HDConfig(**HD_SMALL)
    w, w_b, hw = V.make_weights(cfg, seed=11), V.make_weights(cfg_b, seed=12), H.make_weights(hcfg, seed=13)
    model, model_b, hmodel = ref_model(cfg, w), ref_model(cfg_b, w_b), hd_ref_model(hcfg, hw)
    dm = ref_shim.ref_module("audio_separator.separator.uvr_lib_v5.demucs.demucs")
    for L in list(range(1, 3000, 7)) + list(range(3000, 400001, 997)):
        assert model.valid_length(L) == cfg.valid_length(L) and model.valid_length(model.valid_length(L)) == model.valid_length(L), L
    released = dm.Demucs(sources=["drums", "bass", "other", "vocals"], channels=48)  # the mdx / mdx_extra time-domain geometry
    assert dict(V.param_shapes(V.V3Config(channels=48))) == {k: tuple(v.shape) for k, v in released.state_dict().items()}
    valid_in = np.array([1, 2, 1000, 4095, 44100, 352800, 1764000, 1764001, 1940400])
    valid_ref = np.array([released.valid_length(int(n)) for n in valid_in])
    mix = M.synth_music(3 * N_APPLY, seed=43)

    def fwd(m, c, w_, x, what):
        with torch.no_grad():
            y_ref = m(torch.from_numpy(np.ascontiguousarray(x))).numpy()
        check(f"demucs v3 forward ({what})", y_ref, V.forward(w_, c, x), 2e-5 * max(1.0, np.abs(y_ref).max()))
        return y_ref

    y = fwd(model, cfg, w, mix[None, :, :FWD_LEN], "one chunk")
    yl = fwd(model, cfg, w, mix[None, :, :LONG_LEN], "ragged length, framed BLSTM")
    y2 = fwd(model, cfg, w, np.stack([mix[:, :FWD_LEN], mix[:, FWD_LEN : 2 * FWD_LEN]]), "batch 2")
    check("demucs v3 forward (one chunk = batch entry 0)", y, y2[:1], 1e-6 * max(1.0, np.abs(y).max()))  # stored once, as batch entry 0
    fwd(model_b, cfg_b, w_b, mix[None, :, :FWD_LEN], "second member")

    apply = ref_shim.ref_module("audio_separator.separator.uvr_lib_v5.demucs.apply")
    bag = apply.BagOfModels([model, model_b, hmodel], weights=BAG_WEIGHTS)
    assert [m.segment for m in bag.models] == [SMALL["segment"], SMALL_B["segment"], HD_SMALL["segment"]]  # no bag segment: each member keeps its own
    m2 = torch.from_numpy(mix[:, :N_APPLY])
    mn = (m2 - m2.mean(0).mean()) / m2.mean(0).std()
    members = [(lambda c: V.forward(w, cfg, c), cfg), (lambda c: V.forward(w_b, cfg_b, c), cfg_b), (lambda c: H.forward(hw, hcfg, c), hcfg)]
    out = {}
    for name, split, shifts, seed in (("split", True, 1, 5), ("nosplit", False, 1, 6)):
        random.seed(seed)
        state = random.getstate()
        with torch.no_grad():
            b_ref = apply.apply_model(bag, mn[None], shifts=shifts, split=split, overlap=0.25, device="cpu").numpy()
        random.setstate(state)
        offs = [[random.randint(0, int(0.5 * cfg.samplerate)) for _ in range(shifts)] for _ in members]
        print(f"  {name} shift offsets:", offs)
        got = V.apply_bag(members, BAG_WEIGHTS, mn.numpy()[None], offs, split, 0.25)
        check(f"bag apply_model shifts={shifts} split={split}", b_ref, got, 1e-5 * max(1.0, np.abs(b_ref).max()))
        out[f"bag_{name}_ref"], out[f"bag_{name}_offsets"] = b_ref.astype(np.float32), np.array(offs)
    np.savez_compressed(
        os.path.join(GOLD, "demucs_v3_small.npz"), weights_seed=np.array([11, 12, 13]), mix_seed=43, fwd_len=FWD_LEN, long_len=LONG_LEN, n_apply=N_APPLY,
        bag_weights=np.array(BAG_WEIGHTS), valid_in=valid_in, valid_ref=valid_ref, forward_long_ref=yl.astype(np.float32), forward_b2_ref=y2.astype(np.float32), **out)
    print("wrote tests/golden/demucs_v3_small.npz; oracle pinned: OK")


if __name__ == "__main__":
    main()
