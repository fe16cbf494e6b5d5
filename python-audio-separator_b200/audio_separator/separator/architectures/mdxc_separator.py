"""H100 MDXC architecture plugin (non-Roformer TFC_TDF_net models, e.g. MDX23C-8KFFT-InstVoc_HQ).

Plugin contract of the reference's MDXCSeparator (audio_separator/separator/architectures/mdxc_separator.py:19-228):
ctor `(common_config, arch_config)` with arch keys segment_size / override_model_segment_size / batch_size / overlap /
pitch_shift, `separate(path, custom_output_names)`, `demix(mix) -> {instrument: (2, N)}`.  The chunk loop runs on the GPU
through libb200sep.so (MdxcEngine for TFC_TDF_net checkpoints, RoformerEngine for BS-Roformer and Mel-Band Roformer checkpoints -- the Roformer branch of
demix, mdxc_separator.py:272-343).

arch key `pitch_shift` (semitones, both model families): demix resamples the mix on the GPU from sr to sr * 2**(-s/12), runs the engine on
the result, resamples every stem back by 2**(s/12) and fits it to the mix length (spec_utils.change_pitch_semitones + match_array_shapes,
mdxc_separator.py:230-244, :268-270).  The resampler is b200/resample.py's res_type "sinc_fastest", the reference's choice on Linux
(spec_utils.py:33-37); its choice on macOS / ARM (kaiser_best) is not mirrored.

arch key `b200_sharded` (both model families): one process per GPU under an initialised torch.distributed group (nccl); every rank calls
`separate(path)` on the same file, each track is split by time over the ranks (b200/sharded.py), and rank 0 writes the stem files and returns
their names while the other ranks write nothing and return [].
"""
import os

import numpy as np
import torch

from ..b200.engine import MdxcEngine, TfcNet
from ..b200.resample import match_length, resample
from ..b200.roformer import BSRoformerConfig, BSRoformerNet, MelBandRoformerConfig, RoformerEngine
from ..common_separator import CommonSeparator, load_checkpoint, normalize, tensor_core_math

PITCH_RES_TYPE = "sinc_fastest"  # spec_utils.wav_resolution_float_resampling on Linux


class MDXCSeparator(CommonSeparator):
    def __init__(self, common_config, arch_config):
        super().__init__(config=common_config)
        self.model_data_cfgdict = self.model_data  # the model's YAML as a dict (mdxc_separator.py:60)
        self.segment_size = arch_config.get("segment_size", 256)
        self.override_model_segment_size = arch_config.get("override_model_segment_size", False)
        self.overlap = arch_config.get("overlap", 8)
        self.batch_size = arch_config.get("batch_size", 1)
        self.pitch_shift = arch_config.get("pitch_shift", 0)
        self.process_all_stems = arch_config.get("process_all_stems", True)
        self.is_roformer = bool(self.is_roformer_model)
        self.setup_device(arch_config, "MDXCSeparator", "mdxc_params")
        self.is_primary_stem_main_target = bool(self.model_data_cfgdict["training"].get("target_instrument"))  # :69, both model families
        self._engines = {}  # dim_t -> engine: the chunk length is fixed per engine, and separate() switches it for clips shorter than 10 s (:137-143)
        self.load_model()

    def load_model(self):
        """Replaces TFC_TDF_net(config).load_state_dict(checkpoint) (mdxc_separator.py:76-116)."""
        cfg = self.model_data_cfgdict
        audio, model, training = cfg["audio"], cfg["model"], cfg["training"]
        if self.is_roformer:
            return self._load_roformer(cfg)
        if self.use_autocast:
            self.logger.debug("use_autocast: MDX23C (TFC_TDF_net) keeps full precision; its pair-format kernels have no fp16 mode")
        if model.get("norm") != "InstanceNorm" or model.get("act", "gelu") != "gelu" or list(model.get("scale", [2, 2])) != [2, 2]:
            raise ValueError("the H100 TFC_TDF_net supports norm=InstanceNorm, act=gelu, scale=[2,2] (the MDX23C configuration)")
        self._state = load_checkpoint(self.model_path)
        self._select_engine()

    def _select_engine(self):
        """The engine for the current `override_model_segment_size` (dim_t = segment_size or the model's inference.dim_t, :281-286 / :355-360); built once per dim_t."""
        cfg = self.model_data_cfgdict
        audio, model, training = cfg["audio"], cfg["model"], cfg["training"]
        dim_t = int(self.segment_size if self.override_model_segment_size else cfg["inference"]["dim_t"])
        if dim_t not in self._engines:
            if self.is_roformer:
                eng = RoformerEngine(self.net, dim_t, self.overlap, audio.get("sample_rate", 44100), len(training["instruments"]), max(1, int(self.batch_size)),
                                     dist=self.dist)
                self._engines[dim_t] = (self.net, eng, self.net.forward)
            else:
                targets = 1 if training.get("target_instrument") else len(training["instruments"])
                net = TfcNet(self._state, audio["dim_f"], dim_t, model["num_subbands"], audio.get("num_channels", 2), model["num_scales"], model["num_blocks_per_scale"],
                             model["num_channels"], model["growth"], model["bottleneck_factor"], targets, max_batch=max(1, int(self.batch_size)))
                eng = MdxcEngine(net, audio["n_fft"], audio["hop_length"], audio["dim_f"], dim_t, self.overlap, dist=self.dist)
                self._engines[dim_t] = (net, eng, eng.model_run)
        self.net, self.engine, self.model_run = self._engines[dim_t]

    def _load_roformer(self, cfg):
        """RoformerLoader.load_model (roformer/roformer_loader.py:82-195): BSRoformer(**model section) + load_state_dict."""
        model, training = cfg["model"], cfg["training"]
        if "num_bands" in model:  # roformer_loader.py:_create_mel_band_roformer
            rcfg = MelBandRoformerConfig.from_model_section(model)
        elif "freqs_per_bands" in model:
            rcfg = BSRoformerConfig.from_model_section(model)
        else:
            raise ValueError("Unknown Roformer model type in configuration (neither num_bands nor freqs_per_bands)")
        self.net = BSRoformerNet(rcfg, load_checkpoint(self.model_path), device=self.torch_device, math=tensor_core_math("Roformer", self.use_autocast))
        self._select_engine()

    def _demix_stems(self, orig):
        """(2, N) float32 ndarray -> (n_out, 2, N) ndarray.  Sharded: every rank runs its part of the chunk grid, rank 0 gathers and gets the
        stems, the other ranks get None.  With pitch_shift every rank pitches the whole mix (the resampler is deterministic), the engine runs
        on the pitched length, and rank 0 pitches every stem back and fits it to N (pitch_fix, :230-244)."""
        mix = torch.as_tensor(orig).to(self.torch_device)
        if self.pitch_shift:
            sr_pitched = self.sample_rate * 2 ** (-self.pitch_shift / 12)  # change_pitch_semitones(mix, sr, -pitch_shift) (:268-270)
            mix = resample(mix, self.sample_rate, sr_pitched, PITCH_RES_TYPE)
        part = self.engine.demix_device(mix)
        full = self.engine.gather(part, mix.shape[1])
        if full is None:
            return None
        if self.pitch_shift:
            sr_back = sr_pitched * 2 ** (self.pitch_shift / 12)
            full = torch.stack([match_length(resample(stem, sr_pitched, sr_back, PITCH_RES_TYPE), orig.shape[1]) for stem in full])
        return full.cpu().numpy()

    def demix(self, mix):
        """(2, N) ndarray -> {instrument: (2, N) ndarray} (mdxc_separator.py:272-343, :406-434) or the single target's array; None on the ranks
        other than 0 of a sharded run."""
        orig = np.ascontiguousarray(mix, dtype=np.float32)
        out = self._demix_stems(orig)
        if out is None:
            return None
        if out.shape[0] > 1:  # one row per stem of a multi-stem model
            return dict(zip(self.model_data_cfgdict["training"]["instruments"], out))
        primary = out[0]
        if self.is_primary_stem_main_target:  # single-target models also return the residual as the secondary stem (:452-461)
            return {self.primary_stem_name: primary, self.secondary_stem_name: orig - primary}
        return primary

    def separate(self, audio_file_path, custom_output_names=None):
        self.audio_file_path = audio_file_path
        self.audio_file_base = os.path.splitext(os.path.basename(audio_file_path))[0]
        mix = self.prepare_mix(self.audio_file_path)
        if mix.shape[1] / self.sample_rate < 10.0 and not self.override_model_segment_size:  # :137-143 (the switch is sticky in the reference too)
            self.override_model_segment_size = True
            self.logger.warning(f"Audio duration ({mix.shape[1] / self.sample_rate:.2f}s) is less than 10 seconds.")
            self.logger.warning("Automatically enabling override_model_segment_size for better processing of short audio.")
            self._select_engine()
        mix = normalize(wave=np.array(mix, dtype=np.float32), max_peak=self.normalization_threshold, min_peak=self.amplification_threshold)  # :149
        source = self.demix(mix)
        if source is None:  # sharded, rank != 0: rank 0 holds the stems and writes the files
            return []
        if not isinstance(source, dict):  # a single-source model without a target instrument: only the primary stem is written, as it is (:216-226)
            self.primary_source = source.T
            return self.write_stems([(self.primary_stem_name, self.primary_source)], custom_output_names)
        training = self.model_data_cfgdict["training"]  # (:156-214)
        stem_list = [training["target_instrument"]] if training.get("target_instrument") else list(training["instruments"])
        norm = lambda w: normalize(wave=w, max_peak=self.normalization_threshold, min_peak=self.amplification_threshold).T  # noqa: E731
        if self.process_all_stems and len(stem_list) > 2:  # every stem of a multi-stem model, in the model's order
            return self.write_stems([(name, norm(source[name])) for name in stem_list], custom_output_names)
        self.primary_source, self.secondary_source = norm(source[self.primary_stem_name]), norm(source[self.secondary_stem_name])
        return self.write_stems([(self.secondary_stem_name, self.secondary_source), (self.primary_stem_name, self.primary_source)], custom_output_names)
