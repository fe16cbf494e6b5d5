"""`Separator` facade: same constructor / load_model() / separate() surface as the reference orchestrator
(audio_separator/separator/separator.py:108-257, :830-933, :935-1045), restricted to what the accelerated path
needs.  Model download, ensembles, presets and file-level chunking are out of scope (SURVEY.md section 2, rows 1, 14, 15):
models are looked up in `model_file_dir` only.
"""
import importlib
import json
import logging
import os
import re
import shutil
import tempfile
import time

import numpy as np
import torch

# UVR model_data_new.json entries for the BASELINE models (looked up by MD5 at runtime in the reference, separator.py:786-824)
KNOWN_MODEL_DATA = {
    "UVR-MDX-NET-Inst_HQ_3.onnx": {"compensate": 1.022, "mdx_dim_f_set": 3072, "mdx_dim_t_set": 8, "mdx_n_fft_scale_set": 6144, "primary_stem": "Instrumental"},
    "UVR-MDX-NET-Inst_HQ_5.onnx": {"compensate": 1.010, "mdx_dim_f_set": 2560, "mdx_dim_t_set": 8, "mdx_n_fft_scale_set": 5120, "primary_stem": "Instrumental"},
}


# canonical stem names of the ensemble grouping (separator.py:29-49)
STEM_NAME_MAP = {
    "vocals": "Vocals", "instrumental": "Instrumental", "inst": "Instrumental", "karaoke": "Instrumental", "other": "Other", "no_vocals": "Instrumental",
    "drums": "Drums", "bass": "Bass", "guitar": "Guitar", "piano": "Piano", "synthesizer": "Synthesizer", "strings": "Strings", "woodwinds": "Woodwinds",
    "brass": "Brass", "wind inst": "Wind Inst", "lead vocals": "Lead Vocals", "backing vocals": "Backing Vocals", "primary stem": "Primary Stem",
    "secondary stem": "Secondary Stem",
}
_SLUG_PREFIXES = ("mel_band_roformer_", "melband_roformer_", "bs_roformer_", "model_bs_roformer_", "UVR-MDX-NET-", "UVR_MDXNET_")


class Separator:
    def __init__(self, log_level=logging.INFO, log_formatter=None, model_file_dir="/tmp/audio-separator-models/", output_dir=None, output_format="WAV",
                 output_bitrate=None, normalization_threshold=0.9, amplification_threshold=0.0, output_single_stem=None, invert_using_spec=False,
                 sample_rate=44100, use_soundfile=False, use_autocast=False, use_directml=False, chunk_duration=None,
                 mdx_params=None, vr_params=None, demucs_params=None, mdxc_params=None, ensemble_algorithm=None, ensemble_weights=None,
                 ensemble_preset=None, info_only=False):
        self.logger = logging.getLogger(__name__)
        self.logger.setLevel(log_level)
        self.log_level = log_level
        if not self.logger.hasHandlers():
            h = logging.StreamHandler()
            h.setFormatter(log_formatter or logging.Formatter("%(asctime)s - %(levelname)s - %(module)s - %(message)s"))
            self.logger.addHandler(h)
        self.model_file_dir = os.environ.get("AUDIO_SEPARATOR_MODEL_DIR", model_file_dir)  # separator.py:167
        self.output_dir = output_dir or os.getcwd()
        self.output_format = output_format or "WAV"
        self.output_bitrate = output_bitrate
        if not 0 < normalization_threshold <= 1:
            raise ValueError("The normalization_threshold must be greater than 0 and less than or equal to 1.")
        if not 0 <= amplification_threshold <= 1:
            raise ValueError("The amplification_threshold must be greater than or equal to 0 and less than or equal to 1.")
        self.normalization_threshold, self.amplification_threshold = normalization_threshold, amplification_threshold
        self.output_single_stem, self.invert_using_spec = output_single_stem, invert_using_spec
        self.sample_rate = int(sample_rate)
        if self.sample_rate <= 0 or self.sample_rate > 12800000:
            raise ValueError(f"The sample rate setting is {self.sample_rate} but it must be a non-zero whole number.")
        self.use_soundfile, self.use_autocast = use_soundfile, use_autocast
        if ensemble_preset or chunk_duration:
            raise NotImplementedError("ensemble presets (ensemble_presets.json) / file-level chunking are outside the H100 hot-path scope; pass the model list and algorithm explicitly")
        self.ensemble_algorithm = ensemble_algorithm or "avg_wave"  # separator.py:237-238
        self.ensemble_weights = ensemble_weights
        self.ensemble_preset = None
        self.model_filename = None
        self.model_filenames = []
        self.arch_specific_params = {
            "MDX": {"hop_length": 1024, "segment_size": 256, "overlap": 0.25, "batch_size": 1, "enable_denoise": False, **(mdx_params or {})},
            "VR": {"batch_size": 1, "window_size": 512, "aggression": 5, "enable_tta": False, "enable_post_process": False, "post_process_threshold": 0.2, "high_end_process": False, **(vr_params or {})}, "Demucs": {"segment_size": "Default", "shifts": 2, "overlap": 0.25, "segments_enabled": True, **(demucs_params or {})}, "MDXC": {"segment_size": 256, "override_model_segment_size": False, "batch_size": 1, "overlap": 8, "pitch_shift": 0, **(mdxc_params or {})},
        }
        self.torch_device = self.torch_device_cpu = torch.device("cpu")
        self.torch_device_mps = None
        self.onnx_execution_provider = None
        self.model_instance = None
        self.model_is_uvr_vip = False
        self.model_friendly_name = None
        if not info_only:
            self.setup_accelerated_inferencing_device()

    def setup_accelerated_inferencing_device(self):
        if not torch.cuda.is_available():
            raise RuntimeError("no CUDA device: this build targets H100 (sm_90a) only and has no CPU / MPS / DirectML path")
        self.torch_device = torch.device("cuda", torch.cuda.current_device())
        self.logger.info(f"H100 engine on {torch.cuda.get_device_name(self.torch_device)}")

    def load_model_data(self, model_path):
        if model_path.lower().endswith(".th"):  # a single Demucs package carries its own constructor arguments (demucs/states.py:34-64)
            return {"b200_arch": "Demucs"}
        side = os.path.splitext(model_path)[0] + ".json"
        if os.path.exists(side):
            with open(side, encoding="utf-8") as f:
                return json.load(f)
        for ext in (".yaml", ".yml"):  # MDXC / Demucs models carry a YAML config next to the checkpoint (separator.py:758-777)
            if os.path.exists(os.path.splitext(model_path)[0] + ext):
                import yaml

                with open(os.path.splitext(model_path)[0] + ext, encoding="utf-8") as f:
                    return yaml.safe_load(f)
        name = os.path.basename(model_path)
        if name in KNOWN_MODEL_DATA:
            return dict(KNOWN_MODEL_DATA[name])
        raise ValueError(f"no model parameters for {name}: put a {os.path.basename(side)} (UVR model_data entry) next to the model file")

    def load_model(self, model_filename="UVR-MDX-NET-Inst_HQ_3.onnx"):
        if isinstance(model_filename, (list, tuple)):  # several models = an ensemble: they are loaded one after the other inside separate() (separator.py:839-845)
            if len(model_filename) > 1:
                self.model_filename = list(model_filename)
                self.model_filenames = list(model_filename)
                self.logger.info(f"Multiple models specified for ensembling: {self.model_filenames}")
                return
            model_filename = model_filename[0]
        self.model_filename = model_filename
        self.model_filenames = [model_filename]
        t0 = time.perf_counter()
        model_path = model_filename if os.path.isabs(model_filename) else os.path.join(self.model_file_dir, model_filename)
        if not os.path.isfile(model_path):
            raise FileNotFoundError(f"{model_path} not found (this build does not download models)")
        model_data = self.load_model_data(model_path)
        model_type = model_data.get("b200_arch") or ("VR" if "vr_model_param" in model_data else None) or ("MDXC" if "audio" in model_data and "model" in model_data else (
            "Demucs" if "models" in model_data and model_path.lower().endswith((".yaml", ".yml")) else ("MDX" if model_path.lower().endswith((".onnx", ".npz")) else None)))
        classes = {"MDX": "mdx_separator.MDXSeparator", "VR": "vr_separator.VRSeparator", "Demucs": "demucs_separator.DemucsSeparator", "MDXC": "mdxc_separator.MDXCSeparator"}
        if model_type not in classes:
            raise ValueError(f"Model type not supported (yet): {model_type}")
        common = {
            "logger": self.logger, "log_level": self.log_level, "torch_device": self.torch_device, "torch_device_cpu": self.torch_device_cpu,
            "torch_device_mps": self.torch_device_mps, "onnx_execution_provider": self.onnx_execution_provider,
            "model_name": os.path.splitext(os.path.basename(model_filename))[0], "model_path": model_path, "model_data": model_data,
            "output_format": self.output_format, "output_bitrate": self.output_bitrate, "output_dir": self.output_dir,
            "normalization_threshold": self.normalization_threshold, "amplification_threshold": self.amplification_threshold,
            "output_single_stem": self.output_single_stem, "invert_using_spec": self.invert_using_spec, "sample_rate": self.sample_rate,
            "use_soundfile": self.use_soundfile, "use_autocast": self.use_autocast,
        }
        module_name, class_name = classes[model_type].split(".")
        module = importlib.import_module(f"{__package__}.architectures.{module_name}")
        self.model_instance = getattr(module, class_name)(common_config=common, arch_config=self.arch_specific_params[model_type])
        self.logger.info(f"Loading model completed in {time.perf_counter() - t0:.2f}s")

    def separate(self, audio_file_path, custom_output_names=None):
        if isinstance(self.model_filename, list) and len(self.model_filename) > 1:
            return self._separate_ensemble(audio_file_path, custom_output_names)
        if self.model_instance is None:
            raise ValueError("Initialization failed or model not loaded. Please load a model before attempting to separate.")
        paths = [audio_file_path] if isinstance(audio_file_path, str) else list(audio_file_path)
        outputs = []
        audio_ext = (".wav", ".flac", ".mp3", ".ogg", ".opus", ".m4a", ".aiff", ".ac3")  # separator.py:972
        for path in paths:
            if os.path.isdir(path):  # recursive, audio files only (separator.py:966-979)
                files = [os.path.join(root, f) for root, _, names in os.walk(path) for f in names if f.endswith(audio_ext)]
            else:
                files = [path]
            for f in files:
                try:
                    outputs.extend(self._separate_file(f, custom_output_names))
                except Exception as e:  # per-file errors are logged, not raised (separator.py:978-987)
                    self.logger.error(f"Failed to process file {f}: {e}")
        return outputs

    def _separate_ensemble(self, audio_file_path, custom_output_names=None):
        """Several models on the same file, their stems grouped by canonical stem name and reduced by the Ensembler (separator.py:1242-1412).
        Every model runs on the GPU through its plugin, the intermediate stems go through a temporary directory exactly as in the reference (the file round trip
        quantises them to the input bit depth there too), and the reductions over the model axis run on the GPU (audio_separator/separator/ensembler.py)."""
        from .ensembler import Ensembler

        paths = [audio_file_path] if isinstance(audio_file_path, str) else list(audio_file_path)
        models, output_files = list(self.model_filenames), []
        for path in paths:
            temp_dir = tempfile.mkdtemp(prefix="audio-separator-ensemble-")
            original_output_dir = self.output_dir
            try:
                stems_by_type = {}
                for model_filename in models:
                    self.logger.info(f"Processing with model: {model_filename}")
                    self.load_model(model_filename)
                    self.output_dir = temp_dir
                    self.model_instance.output_dir = temp_dir
                    if self.output_format.lower() == "flac":
                        # lossless either way: WAV intermediates hold the samples the reference's FLAC round trip holds, and need no FLAC reader
                        self.model_instance.output_format = "WAV"
                    try:
                        model_stems = self._separate_file(path, None)  # default "base_(Stem)_model.ext" names: the stem type is parsed from them
                    finally:
                        self.output_dir = original_output_dir
                    names = []
                    for stem_path in model_stems:
                        m = re.search(r"_\(([^)]+)\)", os.path.basename(stem_path))
                        names.append(m.group(1) if m else "Unknown")
                    has_vocal = any("vocal" in n.lower() for n in names)
                    for stem_path, raw in zip(model_stems, names):
                        low = raw.lower()
                        if "vocal" in low and "lead" not in low and "backing" not in low:
                            stem = "Vocals"
                        elif low == "other" and len(names) == 2 and has_vocal:
                            stem = "Instrumental"  # the non-vocal stem of a two-stem model
                        else:
                            stem = STEM_NAME_MAP.get(low, raw.title())
                        stems_by_type.setdefault(stem, []).append(stem_path if os.path.isabs(stem_path) else os.path.join(temp_dir, stem_path))
                ensembler = Ensembler(self.logger, self.ensemble_algorithm, self.ensemble_weights)
                base_name = os.path.splitext(os.path.basename(path))[0]
                writer = self.model_instance
                for stem_name, stem_paths in stems_by_type.items():
                    self.logger.info(f"Ensembling {len(stem_paths)} stems for type: {stem_name}")
                    waves = [writer.prepare_mix(sp) for sp in stem_paths]  # (2, N) float32, the reader the plugins use
                    ens = ensembler.ensemble(waves)
                    if custom_output_names and stem_name in custom_output_names:
                        out_name = custom_output_names[stem_name]
                    else:
                        slugs = []
                        for mf in models:
                            name = os.path.splitext(os.path.basename(mf))[0]
                            for prefix in _SLUG_PREFIXES:
                                if name.startswith(prefix):
                                    name = name[len(prefix):]
                                    break
                            slugs.append(name[:12])
                        out_name = f"{base_name}_({stem_name})_custom_ensemble_{'_'.join(slugs)}"
                    out_path = f"{out_name}.{self.output_format.lower()}"
                    writer.audio_file_path = path
                    writer.output_dir = self.output_dir
                    writer.write_audio(out_path, np.ascontiguousarray(np.asarray(ens).T))
                    output_files.append(os.path.join(self.output_dir, out_path))
            finally:
                self.model_filename, self.model_filenames = list(models), list(models)
                self.model_instance = None
                shutil.rmtree(temp_dir, ignore_errors=True)
        return output_files

    def _separate_file(self, audio_file_path, custom_output_names=None):
        t0 = time.perf_counter()
        out = self.model_instance.separate(audio_file_path, custom_output_names)
        self.model_instance.clear_gpu_cache()
        self.model_instance.clear_file_specific_paths()
        self.logger.info(f"Separation duration: {time.perf_counter() - t0:.2f}s")
        return out
