"""H100 VR architecture plugin (CascadedASPPNet models -- the HP / HP2 / SP "VR arch" v4-v5.0 checkpoints -- and VR 5.1 CascadedNet models).

Plugin contract of the reference's VRSeparator (audio_separator/separator/architectures/vr_separator.py:26-253): ctor
`(common_config, arch_config)` with arch keys batch_size / window_size / aggression / enable_tta / enable_post_process /
post_process_threshold / high_end_process, `separate(path, custom_output_names)` -> [primary, secondary] files.
The multi-band analysis, the patch loop, the mask post-processing and the band synthesis run on the GPU (b200.vr.VREngine).

arch key `b200_sharded`: one process per GPU under an initialised torch.distributed group (nccl); every rank calls `separate(path)` on the same
file, the patches of each track are split over the ranks (b200/sharded.py), and rank 0 writes the stem files and returns their names while the
other ranks write nothing and return [].
"""
import math
import os

import numpy as np

from ..b200 import vr_params
from ..b200.vr import NN_ARCH_SIZES, VR_51_SIZES, VREngine, VRNet, VRNet51
from ..common_separator import CommonSeparator, load_checkpoint, tensor_core_math


class VRSeparator(CommonSeparator):
    def __init__(self, common_config, arch_config):
        super().__init__(config=common_config)
        self.model_capacity = 32, 128
        self.is_vr_51_model = False
        if "nout" in self.model_data and "nout_lstm" in self.model_data:  # vr_separator.py:38-41
            self.model_capacity = self.model_data["nout"], self.model_data["nout_lstm"]
            self.is_vr_51_model = True
        self.model_params = vr_params.load(self.model_data["vr_model_param"], os.path.dirname(self.model_path))
        self.enable_tta = arch_config.get("enable_tta", False)
        self.enable_post_process = arch_config.get("enable_post_process", False)
        self.post_process_threshold = arch_config.get("post_process_threshold", 0.2)
        self.batch_size = arch_config.get("batch_size", 1)
        self.window_size = arch_config.get("window_size", 512)
        self.high_end_process = arch_config.get("high_end_process", False)
        self.aggression_setting = int(arch_config.get("aggression", 5))
        self.aggression = float(self.aggression_setting / 100)
        self.setup_device(arch_config, "VRSeparator", "vr_params")
        self.model_samplerate = self.model_params["sr"]
        self.load_model()

    def load_model(self):
        """nets.determine_model_capacity(bins * 2, nn_arch_size).load_state_dict(checkpoint) (vr_separator.py:166-181)."""
        model_size = math.ceil(os.stat(self.model_path).st_size / 1024)
        nn_arch_size = min(NN_ARCH_SIZES, key=lambda x: abs(x - model_size))
        arch = int(self.model_data.get("b200_nn_architecture", nn_arch_size))  # tests use reduced widths whose file size is off the table
        self.is_vr_51_model = self.is_vr_51_model or arch in VR_51_SIZES  # :175-179
        state = load_checkpoint(self.model_path)
        tc_math = tensor_core_math("VR", self.use_autocast)
        if self.is_vr_51_model:
            self.net = VRNet51(self.model_params["bins"] * 2, self.model_capacity[0], self.model_capacity[1], state, nn_arch_size=arch, device=self.torch_device,
                               math=tc_math)
        else:
            self.net = VRNet(arch, self.model_params["bins"] * 2, state, device=self.torch_device, math=tc_math)
        self.engine = VREngine(self.net, self.model_params, self.window_size, self.aggression_setting, self.primary_stem_name, self.batch_size,
                             dist=self.dist)

    def separate(self, audio_file_path, custom_output_names=None):
        self.audio_file_path = audio_file_path
        self.audio_file_base = os.path.splitext(os.path.basename(audio_file_path))[0]
        wave = self.prepare_mix(audio_file_path)  # the file at 44.1 kHz; librosa.load(sr=<top band's rate>) resamples it (vr_separator.py:273)
        # a model at another rate (e.g. 32 / 48 kHz) gets the mix resampled on the device, and its stems come back at 44.1 kHz (:221-222, :239-240)
        stems = self.engine.separate(np.asarray(wave, dtype=np.float32), enable_tta=bool(self.enable_tta),
                                     post_process_threshold=self.post_process_threshold if self.enable_post_process else None,
                                     high_end_process=bool(self.high_end_process), sr=44100)
        if stems is None:  # sharded, rank != 0: rank 0 holds the stems and writes the files
            return []
        primary, secondary = stems
        self.primary_source, self.secondary_source = primary.T, secondary.T
        if self.output_single_stem and self.output_single_stem.lower() not in (self.primary_stem_name.lower(), self.secondary_stem_name.lower()):
            self.output_single_stem = None  # vr_separator.py:197-199
        return self.write_stems([(self.primary_stem_name, self.primary_source), (self.secondary_stem_name, self.secondary_source)], custom_output_names)
