"""H100 MDX architecture plugin.

Same plugin contract as the reference's MDXSeparator (audio_separator/separator/architectures/mdx_separator.py):
ctor `(common_config, arch_config)`, `separate(path, custom_output_names) -> [filenames]`, `demix`, `run_model`,
`initialize_model_settings`, stem order (secondary file first, then primary, :185-197).  What differs is where the
work runs: the whole per-chunk loop (pad -> STFT -> zero low bins -> ConvTDFNet [+denoise] -> iSTFT -> Hann
overlap-add -> divide -> trim -> *peak -> secondary = mix - compensate*primary) executes on the GPU through
libb200sep.so with all intermediates resident in HBM; the reference crosses host<->device 4x per chunk (:123,:447).
"""
import os

import numpy as np
import torch

from ..b200 import mdx_weights, onnx_reader
from ..b200.engine import MdxEngine, MdxNet
from ..common_separator import CommonSeparator, DeviceStem, load_checkpoint
from ..uvr_lib_v5.stft import STFT


class MDXSeparator(CommonSeparator):
    def __init__(self, common_config, arch_config):
        super().__init__(config=common_config)
        self.segment_size = arch_config.get("segment_size")
        self.overlap = arch_config.get("overlap")
        self.batch_size = arch_config.get("batch_size", 1)
        self.hop_length = arch_config.get("hop_length")
        self.enable_denoise = arch_config.get("enable_denoise")
        self.precision = int(arch_config.get("b200_precision", 1))  # 0 = fp32 SIMT, 1 = bf16x3 split tensor-core path

        self.compensate = self.model_data["compensate"]
        self.dim_f = self.model_data["mdx_dim_f_set"]
        self.dim_t = 2 ** self.model_data["mdx_dim_t_set"]
        self.n_fft = self.model_data["mdx_n_fft_scale_set"]
        self.config_yaml = self.model_data.get("config_yaml", None)

        self.setup_device(arch_config, "MDXSeparator", "mdx_params", missing="onnxruntime / CPU path")
        self.n_bins = self.trim = self.chunk_size = self.gen_size = 0
        self._host_bufs = {}
        self.stft = None
        self.engine = None
        self.load_model()

    # ---- model ------------------------------------------------------------------------------------------
    def load_model(self):
        """Replaces the ort.InferenceSession / onnx2torch branches (mdx_separator.py:108-133): the ONNX initialisers
        are read with a protobuf wire parser and handed to the engine, which folds BatchNorm and lays the weights
        out for its kernels.  `segment_size != dim_t` needs no special case: the TDF layers act on the frequency
        axis only, so the same weights run at any (even) number of frames."""
        path = self.model_path
        if path.lower().endswith(".onnx"):
            state = onnx_reader.load_convtdfnet_state(path)
        elif path.lower().endswith(".npz"):
            state = load_checkpoint(path)
        else:
            raise ValueError(f"unsupported MDX model file {path!r} (expected .onnx or .npz)")
        hp = mdx_weights.infer_hparams_from_state(state)
        if hp["dim_f"] != self.dim_f:
            raise ValueError(f"model_data says mdx_dim_f_set={self.dim_f} but the network's TDF layers were built for dim_f={hp['dim_f']}")
        flat = mdx_weights.flatten_state(state, **hp)
        max_batch = max(1, int(self.batch_size))
        self.net = MdxNet(flat, dim_t=self.segment_size, max_batch=max_batch, precision=self.precision, **hp)
        self.engine = MdxEngine(self.net, self.n_fft, self.hop_length, self.dim_f, self.segment_size, self.overlap, self.compensate, bool(self.enable_denoise), max_batch,
                                dist=self.dist)
        self.model_run = lambda spek: self.net.forward(torch.as_tensor(spek, dtype=torch.float32, device=self.torch_device))

    def initialize_model_settings(self):
        """mdx_separator.py:205-228."""
        self.n_bins = self.n_fft // 2 + 1
        self.trim = self.n_fft // 2
        self.chunk_size = self.hop_length * (self.segment_size - 1)
        self.gen_size = self.chunk_size - 2 * self.trim
        if self.stft is None:
            self.stft = STFT(self.logger, self.n_fft, self.hop_length, self.dim_f, self.torch_device)

    # ---- hot path ---------------------------------------------------------------------------------------
    def run_model(self, mix, is_match_mix=False):
        """(B,2,chunk) tensor -> (B,2,chunk) float32 ndarray, like the reference's run_model (:414-450)."""
        mix = torch.as_tensor(mix, dtype=torch.float32).to(self.torch_device)
        return self.engine.run_model(mix, is_match_mix=is_match_mix).cpu().numpy()

    def demix(self, mix, is_match_mix=False):
        """mix (2,N) float32 ndarray -> source (2,N) float32 ndarray (:293-412)."""
        self.initialize_model_settings()
        mix_dev = torch.as_tensor(np.ascontiguousarray(mix, dtype=np.float32)).to(self.torch_device)
        return self.engine.demix_device(mix_dev, is_match_mix=is_match_mix).cpu().numpy()

    def _pinned(self, name, shape):
        """Page-locked staging buffers, kept between files of the same length (one cudaHostAlloc per size, not per file)."""
        buf = self._host_bufs.get(name)
        if buf is None or tuple(buf.shape) != tuple(shape):
            buf = torch.empty(shape, dtype=torch.float32, pin_memory=True)
            self._host_bufs[name] = buf
        return buf

    def separate_host(self, mix):
        """The array-level body of separate() (mdx_separator.py:152-182) on HOST buffers: mix (2, N) float32 ndarray as prepare_mix returns it ->
        (primary (N, 2), secondary (N, 2)) float32 ndarrays (views of pinned buffers owned by the plugin, valid until the next call).
        One upload, the whole chunk loop on the device, one download per stem."""
        self.initialize_model_settings()
        # a page-locked tensor is uploaded by DMA as it is; a plain ndarray goes through the driver's staged copy (no extra host pass here either way)
        src = mix if isinstance(mix, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(mix, dtype=np.float32))
        N = src.shape[1]
        mix_dev = src.to(self.torch_device, non_blocking=True)
        primary_dev, secondary_dev = self.engine.separate_device(mix_dev, self.normalization_threshold, self.amplification_threshold)
        out_p, out_s = self._pinned("primary", (N, 2)), self._pinned("secondary", (N, 2))
        out_p.copy_(primary_dev, non_blocking=True)
        out_s.copy_(secondary_dev, non_blocking=True)
        torch.cuda.current_stream().synchronize()
        return out_p.numpy(), out_s.numpy()

    def separate_host_shared(self, mix_shared, out_primary, out_secondary):
        """separate_host for the sharded plugin (one process per GPU): the arguments are page-locked host tensors MAPPED BY EVERY RANK -- mix (2, N),
        stems (N, 2).  Each rank uploads the samples its chunks read and downloads the slice of both stems it finalised (b200/sharded.py), so the
        host<->device traffic of one track is spread over all PCIe links.  Returns this rank's (h2d, d2h) bytes."""
        if not self.sharded:
            raise RuntimeError("separate_host_shared needs arch_config['b200_sharded'] and an initialised torch.distributed process group")
        self.initialize_model_settings()
        return self.engine.separate_host(mix_shared, out_primary, out_secondary, self.normalization_threshold, self.amplification_threshold)

    def separate(self, audio_file_path, custom_output_names=None):
        self.audio_file_path = audio_file_path
        self.audio_file_base = os.path.splitext(os.path.basename(audio_file_path))[0]
        mix = self.prepare_mix(self.audio_file_path)
        if self.invert_using_spec:
            raise NotImplementedError("invert_using_spec=True (spec_utils.invert_stem) is not part of the accelerated path yet")
        # device-resident output pipeline: the float stems stay in HBM; write_audio pulls bits/8 bytes per sample (normalise, quantise and pack are kernels)
        self.initialize_model_settings()
        if isinstance(mix, DeviceStem):  # decoded on the GPU (FLAC input): the mix never visits the host
            mix_dev = mix.tensor.to(self.torch_device)
        else:
            mix_dev = torch.from_numpy(np.ascontiguousarray(mix, dtype=np.float32)).to(self.torch_device)
        primary_dev, secondary_dev = self.engine.separate_device(mix_dev, self.normalization_threshold, self.amplification_threshold)
        if not isinstance(self.primary_source, np.ndarray):
            self.primary_source = DeviceStem(primary_dev)
        if not isinstance(self.secondary_source, np.ndarray):
            self.secondary_source = DeviceStem(secondary_dev)
        unwrap = lambda src: src.tensor if isinstance(src, DeviceStem) else src  # noqa: E731
        # secondary stem file first, then primary (:185-197)
        return self.write_stems([(self.secondary_stem_name, unwrap(self.secondary_source)), (self.primary_stem_name, unwrap(self.primary_source))],
                                custom_output_names)
