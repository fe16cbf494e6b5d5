"""H100 Demucs architecture plugin (HTDemucs v4 models and bags: htdemucs, htdemucs_ft, ...; Hybrid Demucs v3: hdemucs_mmi, mdx_extra, ...).

Plugin contract of the reference's DemucsSeparator (audio_separator/separator/architectures/demucs_separator.py:26-195):
ctor `(common_config, arch_config)` with arch keys segment_size / shifts / overlap / segments_enabled,
`separate(path, custom_output_names)`, `demix_demucs(mix) -> (S, 2, N)` with sources 0 and 1 swapped.
Every forward, the shift trick, the segment overlap-add and the bag average run on the GPU (b200.demucs.DemucsEngine).
Time-domain Demucs v1 / v2 packages are not part of this path.

arch key `b200_sharded`: one process per GPU under an initialised torch.distributed group (nccl); every rank calls `separate(path)` on the same
file, the segments of every (model, shift) pass are split by time over the ranks (b200/sharded.py), with rank 0's shift offsets used on every
rank, and rank 0 writes the stem files and returns their names while the other ranks write nothing and return [].
"""
import os
import random
from fractions import Fraction

import numpy as np

from ..b200.demucs import DemucsEngine, HTDemucsNet
from ..b200.demucs_loader import load_demucs
from ..b200.hdemucs import HDemucsConfig, HDemucsNet
from ..common_separator import CommonSeparator, tensor_core_math

DEMUCS_2_SOURCE_MAPPER = {CommonSeparator.INST_STEM: 0, CommonSeparator.VOCAL_STEM: 1}
DEMUCS_4_SOURCE_MAPPER = {CommonSeparator.BASS_STEM: 0, CommonSeparator.DRUM_STEM: 1, CommonSeparator.OTHER_STEM: 2, CommonSeparator.VOCAL_STEM: 3}
DEMUCS_6_SOURCE_MAPPER = {**DEMUCS_4_SOURCE_MAPPER, CommonSeparator.GUITAR_STEM: 4, CommonSeparator.PIANO_STEM: 5}


class DemucsSeparator(CommonSeparator):
    def __init__(self, common_config, arch_config):
        super().__init__(config=common_config)
        self.segment_size = arch_config.get("segment_size", "Default")
        self.shifts = arch_config.get("shifts", 2)
        self.overlap = arch_config.get("overlap", 0.25)
        self.segments_enabled = arch_config.get("segments_enabled", True)
        self.batch_size = int(arch_config.get("batch_size", 4))  # segments per forward (H100 addition; results do not depend on it)
        self.setup_device(arch_config, "DemucsSeparator", "demucs_params")
        self.demucs_source_map = DEMUCS_4_SOURCE_MAPPER
        self.load_model()

    def load_model(self):
        """get_demucs_model(name, repo) + demucs_segments(segment_size, model) (demucs_separator.py:110-114, apply.py:263-300)."""
        models, weights, bag_segment = load_demucs(self.model_path)
        nets = []
        math = tensor_core_math("Demucs", self.use_autocast)
        for cfg, state in models:
            if bag_segment is not None:  # BagOfModels.__init__ (apply.py:58-60)
                cfg.segment = Fraction(bag_segment)
            if self.segment_size != "Default":
                try:
                    cfg.segment = Fraction(int(self.segment_size))  # demucs_segments: sub.segment = int(segment)
                except (TypeError, ValueError):
                    pass
            nets.append((HDemucsNet if isinstance(cfg, HDemucsConfig) else HTDemucsNet)(cfg, state, device=self.torch_device, math=math))
        # segments_enabled=False: apply_model(split=False), one forward over the whole track (HTDemucs raises beyond its training segment, like the reference)
        self.engine = DemucsEngine(nets, bag_weights=weights, overlap=self.overlap, batch_size=self.batch_size, split=bool(self.segments_enabled),
                                   dist=self.dist)

    def demix_demucs(self, mix):
        """(2, N) -> (S, 2, N) (demucs_separator.py:162-195); None on the ranks other than 0 of a sharded run.  The shift offsets are drawn exactly
        where apply_model draws them (`random.randint(0, max_shift)` per shift, per model of the bag, apply.py:207); sharded, every rank draws and then
        takes rank 0's draws, so all ranks run the same passes."""
        max_shift = int(0.5 * self.engine.cfg.samplerate)
        offsets = [[random.randint(0, max_shift) for _ in range(self.shifts)] for _ in self.engine.nets]
        if self.dist is not None:
            box = [offsets]
            self.dist.broadcast_object_list(box, src=0, device=self.torch_device)
            offsets = box[0]
        return self.engine.demix(np.asarray(mix, dtype=np.float32), offsets)

    def separate(self, audio_file_path, custom_output_names=None):
        self.audio_file_path = audio_file_path
        self.audio_file_base = os.path.splitext(os.path.basename(audio_file_path))[0]
        mix = self.prepare_mix(self.audio_file_path)
        source = self.demix_demucs(mix)
        if source is None:  # sharded, rank != 0: rank 0 holds the stems and writes the files
            return []
        self.demucs_source_map = {2: DEMUCS_2_SOURCE_MAPPER, 6: DEMUCS_6_SOURCE_MAPPER}.get(len(source), DEMUCS_4_SOURCE_MAPPER)  # :134-146
        return self.write_stems([(name, source[i].T) for name, i in self.demucs_source_map.items()], custom_output_names)
