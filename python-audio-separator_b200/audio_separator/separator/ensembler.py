"""H100 mirror of the reference's Ensembler (audio_separator/separator/ensembler.py): same constructor `(logger, algorithm, weights)` and
`ensemble(waveforms) -> ndarray`, the reductions over the model axis (and the 2048 / 1024 STFTs of the *_fft and uvr_* algorithms) run on the GPU.
`ensemble_wav` (spec_utils.ensemble_wav: a per-channel pick of the quietest model) is a handful of host comparisons and mirrors the numpy semantics."""
import numpy as np
import torch

from .b200._lib import LAYOUT_CFT, check, lib
from .b200.engine import StftPlan, _ptr, _stream

ALGORITHMS = ("avg_wave", "median_wave", "min_wave", "max_wave", "avg_fft", "median_fft", "min_fft", "max_fft", "uvr_max_spec", "uvr_min_spec", "ensemble_wav")


class Ensembler:
    def __init__(self, logger, algorithm="avg_wave", weights=None):
        self.logger = logger
        self.algorithm = algorithm
        self.weights = weights
        self._plan = None

    def _reduce(self, x, algo, weights=None):
        """x (M, n) cuda -> (n)"""
        out = torch.empty(x.shape[1:], dtype=torch.float32, device=x.device)
        w = torch.as_tensor(np.asarray(weights, dtype=np.float32)).to(x.device) if weights is not None else None
        check(lib.b200sep_ensemble_f32(_ptr(x), x.shape[0], out.numel(), _ptr(w) if w is not None else None, algo, _ptr(out), _stream()), "ensemble_f32")
        return out

    def _stft(self, waves):
        """(M, 2, N) -> planes (M, 4, 1025, 1 + N // 1024): librosa.stft(n_fft=2048, hop_length=1024) per channel (ensembler.py:97-107)"""
        if self._plan is None:
            self._plan = StftPlan(2048, 1024)
        M, _, N = waves.shape
        frames = 1 + N // 1024
        spec = torch.empty((M, 4, 1025, frames), dtype=torch.float32, device=waves.device)
        check(lib.b200sep_stft_forward_ex(self._plan.handle, _ptr(waves), 2 * N, N, 0, M, N, frames, 1024, 1.0, 1025, 0, LAYOUT_CFT, 1, _ptr(spec), _stream()), "stft_forward_ex")
        return spec

    def _istft(self, planes, length):
        """planes (4, 1025, frames) -> (2, length): librosa.istft(hop_length=1024, length=length) (ensembler.py:109-122)"""
        frames = planes.shape[2]
        wave = torch.empty((2, length), dtype=torch.float32, device=planes.device)
        work = torch.empty(lib.b200sep_stft_inverse_work_floats(self._plan.handle, 1, frames, 1025, LAYOUT_CFT), dtype=torch.float32, device=planes.device)
        check(lib.b200sep_stft_inverse_ex(self._plan.handle, _ptr(planes), 1, frames, 1025, LAYOUT_CFT, length, 1024, 0, 1.0, _ptr(wave), _ptr(work), _stream()), "stft_inverse_ex")
        return wave

    @staticmethod
    def _ensemble_wav(waveforms, split_size=240):
        """spec_utils.ensemble_wav (spec_utils.py:1245-1266): every waveform is np.array_split into 240 parts ALONG ITS FIRST AXIS -- for the (channels, length)
        arrays the Separator passes that is the channel axis, so parts 0..channels-1 are one channel row each and the rest are empty -- and for every part the
        waveform with the lowest mean |x| is taken.  A few comparisons per file: host arithmetic, same numpy semantics (an empty part's mean is nan and
        argmin then picks the first waveform)."""
        parts = [np.array_split(np.asarray(w), split_size) for w in waveforms]
        out = []
        with np.errstate(invalid="ignore", divide="ignore"):
            import warnings

            with warnings.catch_warnings():
                warnings.simplefilter("ignore", RuntimeWarning)
                for k in range(split_size):
                    means = [np.abs(p[k]).mean() for p in parts]
                    out.append(parts[int(np.argmin(means))][k])
        return np.concatenate(out)

    def ensemble(self, waveforms):
        """waveforms: list of (channels, length) arrays -> (channels, length) (ensembler.py:18-92)"""
        if not waveforms:
            return None
        if len(waveforms) == 1:
            return waveforms[0]
        if self.algorithm not in ALGORITHMS:
            raise ValueError(f"Unknown ensemble algorithm: {self.algorithm}")
        if self.algorithm == "ensemble_wav":
            if any(w.shape[0] != waveforms[0].shape[0] for w in waveforms):
                raise ValueError("All waveforms must have the same number of channels for ensembling.")
            n = max(w.shape[1] for w in waveforms)  # zero-padded to the longest first (ensembler.py:27-29)
            return self._ensemble_wav([np.pad(w, ((0, 0), (0, n - w.shape[1]))) if w.shape[1] < n else w for w in waveforms])
        if not torch.cuda.is_available():
            raise RuntimeError("Ensembler (H100 build) needs a CUDA device: there is no CPU path in this package")
        num_channels = waveforms[0].shape[0]
        if any(w.shape[0] != num_channels for w in waveforms):
            raise ValueError("All waveforms must have the same number of channels for ensembling.")
        if len(waveforms) > 16:
            raise ValueError("the accelerated ensembler handles at most 16 models")
        max_length = max(w.shape[1] for w in waveforms)
        host = np.zeros((len(waveforms), num_channels, max_length), np.float32)
        for i, w in enumerate(waveforms):
            host[i, :, : w.shape[1]] = w
        if self.weights is None:
            weights = np.ones(len(waveforms))
        else:
            weights = np.array(self.weights)
            if len(weights) != len(waveforms):
                self.logger.warning(f"Number of weights ({len(weights)}) does not match number of waveforms ({len(waveforms)}). Using equal weights.")
                weights = np.ones(len(waveforms))
            weights_sum = np.sum(weights)
            if not np.all(np.isfinite(weights)) or not np.isfinite(weights_sum) or weights_sum == 0:
                self.logger.warning(f"Weights {self.weights} contain non-finite values or sum to zero. Falling back to equal weights.")
                weights = np.ones(len(waveforms))
        if self.algorithm not in ("avg_wave", "avg_fft") and self.weights is not None and not np.all(weights == weights[0]):
            self.logger.warning(f"Weights are ignored for algorithm {self.algorithm}")
        x = torch.from_numpy(host).cuda()
        M = x.shape[0]
        wave_algo = {"avg_wave": 0, "median_wave": 1, "min_wave": 2, "max_wave": 3}
        if self.algorithm in wave_algo:
            return self._reduce(x.view(M, -1), wave_algo[self.algorithm], weights).view(num_channels, max_length).cpu().numpy()
        # spectral algorithms work on stereo STFTs (mono input is duplicated, ensembler.py:98-101)
        st = x if num_channels == 2 else x.expand(M, 2, max_length).contiguous()
        if num_channels not in (1, 2):
            raise ValueError("spectral ensembling handles mono or stereo stems")
        specs = self._stft(st)
        P = specs.shape[2] * specs.shape[3]
        if self.algorithm in ("avg_fft", "median_fft"):
            ens = self._reduce(specs.view(M, -1), 0 if self.algorithm == "avg_fft" else 1, weights).view(4, specs.shape[2], specs.shape[3])
        else:
            take_max = self.algorithm in ("max_fft", "uvr_max_spec")
            last = self.algorithm.startswith("uvr_")
            ens = torch.empty((4, specs.shape[2], specs.shape[3]), dtype=torch.float32, device=x.device)
            check(lib.b200sep_ensemble_spec_abs(_ptr(specs), M, P, int(take_max), int(last), _ptr(ens), _stream()), "ensemble_spec_abs")
        if self.algorithm.startswith("uvr_"):  # spectrogram_to_wave_no_mp: librosa.istft without `length` -> hop * (frames - 1) samples (spec_utils.py:538-544)
            return self._istft(ens, 1024 * (specs.shape[3] - 1)).cpu().numpy()[:num_channels]
        wave = self._istft(ens, max_length).cpu().numpy()
        return wave[:1, :] if num_channels == 1 else wave
