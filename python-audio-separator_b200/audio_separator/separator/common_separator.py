"""Base class contract shared by the H100 architecture plugins.

Mirrors what `Separator` and the plugins rely on from the reference's CommonSeparator
(audio_separator/separator/common_separator.py:57-157 config/stem naming, :217-282 prepare_mix,
:284-451 write_audio, :453-507 cache + output paths).  Audio decode is NOT part of the accelerated
path (SURVEY.md section 2, row 2): 16-32-bit integer PCM WAV goes through the stdlib `wave` module, FLAC (recognised
by content) is decoded on the GPU (b200/flac.py) into a DeviceStem, as are the other uncompressed WAV, RF64, AIFF and AIFF-C files (b200/pcm_reader.py),
anything else goes through soundfile/librosa when those wheels are installed.  Output: WAV through `wave`, FLAC encoded on the GPU
(b200/flac.py), anything else through soundfile.
"""
import gc
import os
import re
import wave as _wave

import numpy as np
import torch

_PAIR = {"Vocals": "Instrumental", "Instrumental": "Vocals", "lead_only": "backing_only", "backing_only": "lead_only", "Primary Stem": "Secondary Stem"}


def normalize(wave, max_peak=1.0, min_peak=None):
    """spec_utils.normalize (uvr_lib_v5/spec_utils.py:99-115), in place like the reference."""
    maxv = np.abs(wave).max()
    if maxv > max_peak:
        wave *= max_peak / maxv
    elif min_peak is not None and maxv < min_peak:
        wave *= min_peak / maxv
    return wave


# Architectures whose PyTorch linears, convolutions and attention products torch.autocast("cuda") runs in fp16 in the reference (use_autocast=True):
# here their tensor-core launches take the same precision (B200SEP_MATH_FP16).  MDX-Net runs in ONNX Runtime in the reference, which autocast does
# not touch, so it keeps full precision; MDX23C does too, because its pair-format kernels have no fp16 activation storage format yet.
AUTOCAST_FP16_ARCHS = ("Demucs", "VR", "Roformer")


def tensor_core_math(arch: str, use_autocast) -> int:
    """The math mode (b200._lib.MATH_*) of the tensor-core launches of architecture `arch` ("MDX", "MDX23C", "Demucs", "VR", "Roformer")."""
    from .b200._lib import MATH_BF16X3, MATH_FP16

    return MATH_FP16 if use_autocast and arch in AUTOCAST_FP16_ARCHS else MATH_BF16X3


def load_checkpoint(path) -> dict:
    """Model weights -> {name: ndarray}: a `.npz` as stored, anything else through torch.load(weights_only=True) as float32 arrays (the
    `state_dict` entry of a training checkpoint, the mapping itself otherwise)."""
    if path.lower().endswith(".npz"):
        with np.load(path) as z:
            return {k: z[k] for k in z.files}
    sd = torch.load(path, map_location="cpu", weights_only=True)
    return {k: v.float().numpy() for k, v in sd.get("state_dict", sd).items()}


class DeviceStem:
    """A float stem that lives in HBM.  `primary_source` / `secondary_source` of a plugin hold these after separate(); np.asarray(stem) downloads it
    (once) for code that expects the reference's host arrays, while write_audio consumes the tensor directly."""

    def __init__(self, tensor):
        self.tensor = tensor
        self._host = None

    @property
    def shape(self):
        return tuple(self.tensor.shape)

    def __array__(self, dtype=None, copy=None):
        if self._host is None:
            self._host = self.tensor.detach().cpu().numpy()
        return self._host if dtype is None else self._host.astype(dtype, copy=False)


class CommonSeparator:
    VOCAL_STEM, INST_STEM, OTHER_STEM, BASS_STEM, DRUM_STEM = "Vocals", "Instrumental", "Other", "Bass", "Drums"
    GUITAR_STEM, PIANO_STEM, PRIMARY_STEM, SECONDARY_STEM, NO_STEM = "Guitar", "Piano", "Primary Stem", "Secondary Stem", "No "
    STEM_PAIR_MAPPER = _PAIR
    _mix_slice = None  # separate_mix: the samples prepare_mix hands to separate() in place of the file's
    _collected = None  # separate_mix(collect=True): the (stem_name, stem) pairs write_stems collects instead of writing

    _CONFIG_KEYS = (
        "logger", "log_level", "torch_device", "torch_device_cpu", "torch_device_mps", "onnx_execution_provider", "model_name", "model_path",
        "model_data", "output_dir", "output_format", "output_bitrate", "normalization_threshold", "amplification_threshold", "enable_denoise",
        "output_single_stem", "invert_using_spec", "sample_rate", "use_soundfile", "use_autocast",
    )

    def __init__(self, config):
        for key in self._CONFIG_KEYS:
            setattr(self, key, config.get(key))
        self.model_data = self.model_data or {}
        self.roformer_loader = None
        name_l, path_l = (self.model_name or "").lower(), (self.model_path or "").lower()
        self.is_roformer_model = bool(self.model_data.get("is_roformer")) or "roformer" in name_l or "roformer" in path_l
        self.input_bit_depth = self.input_subtype = None
        instruments = (self.model_data.get("training") or {}).get("instruments") or []
        if instruments:  # common_separator.py:103-121
            target = self.model_data["training"].get("target_instrument")
            swap = bool(target) and len(instruments) >= 2 and instruments[0] != target and instruments[1] == target
            self.primary_stem_name = instruments[1] if swap else instruments[0]
            self.secondary_stem_name = instruments[0] if swap else (instruments[1] if len(instruments) > 1 else self.secondary_stem(instruments[0]))
        else:
            self.primary_stem_name = self.model_data.get("primary_stem", "Vocals")
            self.secondary_stem_name = self.secondary_stem(self.primary_stem_name)
        self.is_karaoke = self.model_data.get("is_karaoke", False)
        self.is_bv_model = self.model_data.get("is_bv_model", False)
        self.bv_model_rebalance = self.model_data.get("is_bv_model_rebalanced", 0)
        self.cached_sources_map = {}
        self.clear_file_specific_paths()

    def secondary_stem(self, primary_stem):
        primary_stem = primary_stem or self.NO_STEM
        if primary_stem in _PAIR:
            return _PAIR[primary_stem]
        return primary_stem.replace(self.NO_STEM, "") if self.NO_STEM in primary_stem else f"{self.NO_STEM}{primary_stem}"

    def separate(self, audio_file_path, custom_output_names=None):
        raise NotImplementedError

    def setup_device(self, arch_config, name, params_key, missing="CPU path"):
        """Sets `torch_device` (the current CUDA device), `sharded` (arch key `b200_sharded`: one process per GPU under an initialised
        torch.distributed group, nccl, every track split by time over the ranks) and `dist` (the torch.distributed module when sharded, else
        None).  `name` (the plugin's class), `params_key` (its *_params argument) and `missing` (what this package lacks) word the errors."""
        self.sharded = bool(arch_config.get("b200_sharded", False))
        if not torch.cuda.is_available():
            raise RuntimeError(f"{name} (H100 build) needs a CUDA device: there is no {missing} in this package")
        self.dist = None
        if self.sharded:
            import torch.distributed as dist

            if not dist.is_initialized():
                raise RuntimeError(f"{params_key}['b200_sharded'] needs torch.distributed to be initialised (backend nccl, one process per GPU)")
            self.dist = dist
        self.torch_device = torch.device("cuda", torch.cuda.current_device())

    def get_roformer_loading_stats(self):
        return {}

    # ---- input ----------------------------------------------------------------------------------------
    def separate_mix(self, audio_file_path, mix, custom_output_names=None, collect=False):
        """separate(audio_file_path, custom_output_names) run on `mix` -- a (C, n) CUDA tensor or DeviceStem holding that file's samples, or one
        chunk of them, decoded by the caller -- instead of a decode of the file; input_bit_depth stays as the caller's decode set it.  Returns
        what separate() returns; with `collect`, the stems are not written and the plugin's (stem_name, stem) pairs come back instead, in its
        order and after its output_single_stem filter, each peak-normalised on the device ((n, 2) float32 CUDA) or None when near-silent."""
        self._mix_slice, self._collected = mix, ([] if collect else None)
        try:
            out = self.separate(audio_file_path, custom_output_names)
            return self._collected if collect else out
        finally:
            self._mix_slice = self._collected = None

    def prepare_mix(self, mix):
        """path, (N, C) ndarray or mix slice ((C, N) CUDA tensor / DeviceStem) -> float32 (2, N) (common_separator.py:217-282).  Inside
        separate_mix the path separate() passes stands for the caller's samples.  A mix slice leaves input_bit_depth as it is."""
        if self._mix_slice is not None and isinstance(mix, str):
            mix = self._mix_slice
        if isinstance(mix, DeviceStem):
            mix = mix.tensor
        if isinstance(mix, torch.Tensor):
            return self._device_mix(f"{self.audio_file_path} (mix slice)", mix.to(self.torch_device).float().contiguous())
        if isinstance(mix, np.ndarray):
            if self.input_bit_depth is None:
                self.input_bit_depth, self.input_subtype = 16, "PCM_16"
            data = mix.T
        else:
            data = self._read_audio(mix)
            if isinstance(data, torch.Tensor):
                return self._device_mix(mix, data)
            if not np.any(data):
                raise ValueError(f"Audio file {mix} is empty or not valid")
        if data.ndim == 1:
            data = np.asfortranarray([data, data])
        return data

    def _device_mix(self, path, data):
        """A decoded (C, N) CUDA mix -> DeviceStem of (2, N): the "empty or not valid" check by the b200sep_absmax kernel, mono as two equal rows."""
        from .b200._lib import check, lib

        peak = torch.empty(1, dtype=torch.float32, device=data.device)
        check(lib.b200sep_absmax(data.data_ptr(), data.numel(), peak.data_ptr(), torch.cuda.current_stream(data.device).cuda_stream), "absmax")
        if data.numel() == 0 or float(peak.item()) == 0.0:
            raise ValueError(f"Audio file {path} is empty or not valid")
        if data.shape[0] == 1:
            data = data.expand(2, -1).contiguous()
        return DeviceStem(data)

    def _read_flac(self, path):
        """FLAC decoded on the GPU (b200/flac.py): (C, N) float32 CUDA tensor, C = min(channels, 2)."""
        from .b200 import flac

        with open(path, "rb") as f:
            data = f.read()
        info, _, _ = flac.parse(data)
        if info["sample_rate"] != self.sample_rate:
            return None
        depth, subtype = flac.input_bit_depth(info["bps"]) if info["bps"] <= 24 else (None, None)
        mix, info = flac.decode(data, self.torch_device if self.torch_device is not None and self.torch_device.type == "cuda" else "cuda")
        if info["total_samples"] and info["total_samples"] != info["n_samples"]:
            self.logger.warning(f"{path}: STREAMINFO gives {info['total_samples']} samples, the frames hold {info['n_samples']}")
        self.input_bit_depth, self.input_subtype = depth, subtype
        return mix

    def _read_pcm(self, path):
        """Uncompressed WAV / RF64 / AIFF / AIFF-C (recognised by content) decoded on the GPU (b200/pcm_reader.py): (C, N) float32 CUDA tensor,
        C = min(channels, 2); None for another container, another sample rate or a compressed payload (those take the librosa path)."""
        from .b200 import pcm_reader

        with open(path, "rb") as f:
            if not pcm_reader.is_pcm_container(f.read(12)):
                return None
            f.seek(0)
            data = f.read()
        try:
            info = pcm_reader.parse(data)
        except NotImplementedError:
            return None
        if info["sample_rate"] != self.sample_rate:
            return None
        for w in info["warnings"]:
            self.logger.warning(f"{path}: {w}")
        depth, subtype = pcm_reader.input_bit_depth(info)
        if subtype == "PCM_U8":
            self.logger.warning(f"Unknown audio subtype {subtype}, defaulting to 16-bit output")
        mix, _ = pcm_reader.decode(data, self.torch_device if self.torch_device is not None and self.torch_device.type == "cuda" else "cuda")
        self.input_bit_depth, self.input_subtype = depth, subtype
        return mix

    def _read_audio(self, path):
        from .b200 import flac

        if flac.is_flac(path):
            mix = self._read_flac(path)
            if mix is not None:
                return mix
        elif path.lower().endswith(".wav"):
            try:
                with _wave.open(path, "rb") as wf:
                    ch, width, sr, n = wf.getnchannels(), wf.getsampwidth(), wf.getframerate(), wf.getnframes()
                    raw = wf.readframes(n)
                if sr == self.sample_rate and width in (2, 3, 4):
                    self.input_bit_depth, self.input_subtype = width * 8, f"PCM_{width * 8}"
                    if width == 3:
                        b = np.frombuffer(raw, dtype=np.uint8).reshape(-1, 3).astype(np.int32)
                        ints = ((b[:, 0] | (b[:, 1] << 8) | (b[:, 2] << 16)) << 8) >> 8
                    else:
                        ints = np.frombuffer(raw, dtype={2: "<i2", 4: "<i4"}[width]).astype(np.int64)
                    data = (ints.astype(np.float64) / float(1 << (8 * width - 1))).astype(np.float32).reshape(-1, ch).T
                    return data[0] if ch == 1 else np.ascontiguousarray(data[:2])
            except _wave.Error:
                pass
        mix = self._read_pcm(path)
        if mix is not None:
            return mix
        try:
            import librosa
            import soundfile as sf
        except ImportError as e:
            raise RuntimeError(f"cannot decode {path}: only PCM WAV at {self.sample_rate} Hz is supported without librosa/soundfile") from e
        sub = sf.info(path).subtype
        self.input_subtype = sub
        self.input_bit_depth = 24 if "24" in sub else 32 if ("32" in sub or "FLOAT" in sub or "DOUBLE" in sub) else 16
        data, _ = librosa.load(path, mono=False, sr=self.sample_rate)
        return data

    # ---- output ---------------------------------------------------------------------------------------
    def final_process(self, stem_path, source, stem_name):
        self.write_audio(stem_path, source)
        return {stem_name: source}

    def write_stems(self, stems, custom_output_names):
        """Writes the (stem_name, source) pairs in their order -- only the one named `output_single_stem` (any case) when that is set -- and returns
        the paths written.  The path of the primary / secondary stem is also kept in primary_stem_output_path / secondary_stem_output_path."""
        paths = []
        for name, source in stems:
            if self.output_single_stem and self.output_single_stem.lower() != name.lower():
                continue
            if self._collected is not None:
                self._collected.append((name, self._normalized_on_device(self._cuda_stem(source))))
                continue
            path = self.get_stem_output_path(name, custom_output_names)
            self.logger.info(f"Saving {name} stem to {path}...")
            self.final_process(path, source, name)
            if name == self.primary_stem_name:
                self.primary_stem_output_path = path
            elif name == self.secondary_stem_name:
                self.secondary_stem_output_path = path
            paths.append(path)
        return paths

    def _output_bits(self):
        """Output sample width follows the input file (common_separator.py:322-324); 16 bits when unknown."""
        return self.input_bit_depth if self.input_bit_depth in (16, 24, 32) else 16

    @staticmethod
    def _cuda_stem(source):
        """A float stem as a float32 CUDA tensor (a host array is uploaded)."""
        if not (isinstance(source, torch.Tensor) and source.is_cuda):
            source = torch.as_tensor(np.ascontiguousarray(source, dtype=np.float32), device="cuda")
        return source.float()

    def _normalized_on_device(self, stem):
        """spec_utils.normalize of a CUDA stem with the b200sep_absmax / _normalize kernels; None (with the reference's warning) for a near-silent stem."""
        from .b200.engine import normalize_scale, peak_normalize

        norm, peak = peak_normalize(stem.contiguous(), self.normalization_threshold, self.amplification_threshold)
        pk = float(peak.item())
        if pk * normalize_scale(pk, self.normalization_threshold, self.amplification_threshold) < 1e-6:
            self.logger.warning("Warning: stem_source array is near-silent or empty.")
            return None
        return norm

    def pcm_bytes(self, stem_source):
        """(N, 2) float stem -> (bits, interleaved little-endian PCM bytes) at the input's bit depth, or None for a near-silent stem.
        A CUDA tensor never leaves the device as floats: peak, normalisation, quantisation and byte packing are kernels (b200sep_absmax / _normalize /
        _to_pcm_bytes), the host receives bits/8 bytes per sample.  A host array takes the numpy path of the reference."""
        bits = self._output_bits()
        via16 = not self.use_soundfile  # write_audio_pydub quantises to int16 first; write_audio_soundfile converts the floats (:322-336 / :391-451)
        if isinstance(stem_source, torch.Tensor) and stem_source.is_cuda:
            norm = self._normalized_on_device(stem_source)
            if norm is None:
                return None
            return bits, self.pack_pcm(norm, bits).tobytes()
        if isinstance(stem_source, np.ndarray) and stem_source.dtype == np.int16:
            q = stem_source.reshape(-1).astype(np.int64)
            via16 = True
        else:
            s = normalize(np.array(stem_source, dtype=np.float32, copy=True), self.normalization_threshold, self.amplification_threshold)
            if np.max(np.abs(s)) < 1e-6:
                self.logger.warning("Warning: stem_source array is near-silent or empty.")
                return None
            s = np.ascontiguousarray(s).reshape(-1)
            if via16:
                q = (s * 32767).astype(np.int16).astype(np.int64)
            elif bits == 32:
                q = np.clip(np.rint(s.astype(np.float64) * 2147483648.0), -2147483648.0, 2147483647.0).astype(np.int64)
            else:
                q = np.rint(s * np.float32((1 << (bits - 1)) - 1)).astype(np.int64)
        if via16:
            q = q << (bits - 16)
        if bits == 16:
            return bits, q.astype("<i2").tobytes()
        if bits == 32:
            return bits, q.astype("<i4").tobytes()
        b4 = q.astype("<i4").view(np.uint8).reshape(-1, 4)
        return bits, np.ascontiguousarray(b4[:, :3]).tobytes()

    def pack_pcm(self, norm, bits):
        """A peak-normalised CUDA stem -> its interleaved little-endian PCM at `bits` bits as a host uint8 array, quantised on the device by the
        writer's rule (b200sep_to_pcm_bytes; int16 first unless use_soundfile)."""
        from .b200._lib import check, lib

        out = torch.empty(norm.numel() * bits // 8, dtype=torch.uint8, device=norm.device)
        check(lib.b200sep_to_pcm_bytes(norm.data_ptr(), norm.numel(), bits, int(not self.use_soundfile), out.data_ptr(),
                                       torch.cuda.current_stream().cuda_stream), "to_pcm_bytes")
        return out.cpu().numpy()

    def write_flac(self, stem_path, stem_source):
        """`.flac` output encoded on the GPU (b200/flac.py).  A CUDA stem never leaves the device as PCM; a host array is uploaded first.  The stored
        samples are the WAV writer's at the input bit depth, at the stream sample size of the reference's writer (flac.stream_bps)."""
        from .b200 import flac

        if isinstance(stem_source, np.ndarray) and stem_source.dtype == np.int16:
            raise TypeError("FLAC output takes float stems")
        norm = self._normalized_on_device(self._cuda_stem(stem_source))
        if norm is None:
            return
        bits = self._output_bits()
        bps = flac.stream_bps(bits, bool(self.use_soundfile))
        if self.output_dir:
            os.makedirs(self.output_dir, exist_ok=True)
            stem_path = os.path.join(self.output_dir, stem_path)
        if bps is None:
            self.logger.error(f"Error exporting audio file: libsndfile has no {bits}-bit FLAC subtype, {stem_path} not written")
            return
        data = flac.encode(norm, bits, not self.use_soundfile, bps, int(self.sample_rate))
        with open(stem_path, "wb") as f:
            f.write(data)

    def write_audio(self, stem_path, stem_source):
        if stem_path.lower().endswith(".flac"):
            return self.write_flac(stem_path, stem_source)
        packed = self.pcm_bytes(stem_source)
        if packed is None:
            return
        bits, data = packed
        if self.output_dir:
            os.makedirs(self.output_dir, exist_ok=True)
            stem_path = os.path.join(self.output_dir, stem_path)
        if stem_path.lower().endswith(".wav"):
            with _wave.open(stem_path, "wb") as wf:
                wf.setnchannels(2)
                wf.setsampwidth(bits // 8)
                wf.setframerate(int(self.sample_rate))
                wf.writeframes(data)
            return
        try:
            import soundfile as sf
        except ImportError as e:
            raise RuntimeError(f"writing {stem_path}: only WAV output is available without soundfile/pydub") from e
        dt = {16: "<i2", 32: "<i4"}.get(bits)
        if dt is None:  # 24-bit: hand libsndfile int32 with the sample in the top three bytes
            a = np.frombuffer(data, dtype=np.uint8).reshape(-1, 3)
            pcm = (np.concatenate([np.zeros((a.shape[0], 1), np.uint8), a], axis=1).view("<i4")).reshape(-1, 2)
        else:
            pcm = np.frombuffer(data, dtype=dt).reshape(-1, 2)
        sf.write(stem_path, pcm, self.sample_rate, subtype=f"PCM_{bits}")

    def clear_gpu_cache(self):
        gc.collect()
        if torch.cuda.is_available():
            torch.cuda.empty_cache()

    def clear_file_specific_paths(self):
        self.audio_file_path = self.audio_file_base = None
        self.primary_source = self.secondary_source = None
        self.primary_stem_output_path = self.secondary_stem_output_path = None

    def cached_sources_clear(self):
        self.cached_sources_map = {}

    @staticmethod
    def sanitize_filename(filename):
        return re.sub(r"_+", "_", re.sub(r'[<>:"/\\|?*]', "_", filename)).strip("_. ")

    def get_stem_output_path(self, stem_name, custom_output_names):
        ext = self.output_format.lower()
        if custom_output_names:
            lowered = {k.lower(): v for k, v in custom_output_names.items()}
            if stem_name.lower() in lowered:
                return f"{self.sanitize_filename(lowered[stem_name.lower()])}.{ext}"
        parts = [self.sanitize_filename(x) for x in (self.audio_file_base, stem_name, self.model_name)]
        return f"{parts[0]}_({parts[1]})_{parts[2]}.{ext}"
