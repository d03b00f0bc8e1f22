"""Drop-in for ``microwakeword.audio.spectrograms.SpectrogramGeneration`` (reference: microwakeword/audio/spectrograms.py:23-113,
SURVEY.md section 8 row f-3): spectrogram features for a stream of (augmented) audio clips, optionally split into
non-overlapping segments or slid into overlapping copies, ready for ``RaggedMmap.from_generator`` (notebook :286-310).

What changes is only WHERE the features are computed: the reference runs one clip at a time through the native frontend
(:84-86, its slowest offline step); here clips are pulled from the clip generator in batches and every batch -- clips of
different lengths -- goes through ONE launch of the GPU frontend (audio_utils.generate_features_for_clips).  Clip retrieval
(`Clips`) and augmentation (`Augmentation`) are training-data preparation and stay whatever object the caller passes
(SURVEY.md section 2: out of scope); only their generator surface is used.
"""

from __future__ import annotations

import itertools
import os

import numpy as np

from .audio_utils import generate_features_for_clip, generate_features_for_clips


def split_or_slide(spectrogram: np.ndarray, step_ms: int = 20, split_spectrogram_duration_s=None, slide_frames=None):
    """The post-processing of one clip's spectrogram (spectrograms.py:88-113) as a list of arrays.

    split: segments of L = int(duration / (step_ms / 1000)) rows starting at rows 20, 20 + L, ... (the first 20 feature
           windows are dropped), only if the spectrogram has MORE than L + 20 rows, else the whole spectrogram (:88-102);
    slide: `slide_frames` copies of length T - slide_frames + 1 starting at rows 0 .. slide_frames - 1 (:103-111);
    neither: the spectrogram itself.  Returned arrays are views like the reference's sliding_window_view outputs."""
    if split_spectrogram_duration_s is not None:
        length = int(split_spectrogram_duration_s / (step_ms / 1000))
        if spectrogram.shape[0] > length + 20:
            n_windows = spectrogram.shape[0] - length + 1                    # sliding_window_view(...)[20::length]
            # np.squeeze as the reference applies it (:100-101): a one-row segment comes out 1-D
            return [np.squeeze(spectrogram[s:s + length]) for s in range(20, n_windows, length)]
        return [spectrogram]
    if slide_frames is not None:
        length = spectrogram.shape[0] - slide_frames + 1
        if length < 0:
            raise ValueError("window shape cannot be larger than input array shape")       # what sliding_window_view raises
        return [np.squeeze(spectrogram[i:i + length]) for i in range(slide_frames)]
    return [spectrogram]


class SpectrogramGeneration:
    """Same constructor and methods as the reference class (spectrograms.py:23-49).  `batch_clips` (new, optional) is how
    many clips share one frontend launch."""

    def __init__(self, clips, augmenter=None, step_ms: int = 20, split_spectrogram_duration_s=None, slide_frames=None,
                 batch_clips: int = 256, device: int = 0):
        self.clips = clips
        self.augmenter = augmenter
        self.step_ms = step_ms
        self.split_spectrogram_duration_s = split_spectrogram_duration_s
        self.slide_frames = slide_frames
        self.batch_clips = max(int(batch_clips), 1)
        self.device = device

    def get_random_spectrogram(self):
        clip = self.clips.get_random_clip()
        if self.augmenter is not None:
            clip = self.augmenter.augment_clip(clip)
        return generate_features_for_clip(clip, self.step_ms, device=self.device)

    def spectrogram_generator(self, random=False, max_clips=None, **kwargs):
        """Yields 2-D float32 spectrograms in the order the reference would (spectrograms.py:61-113)."""
        if random:
            clip_generator = self.clips.random_audio_generator(max_clips=max_clips) if max_clips is not None else self.clips.random_audio_generator()
        else:
            clip_generator = self.clips.audio_generator(**kwargs)
        if self.augmenter is not None:
            clip_generator = self.augmenter.augment_generator(clip_generator)
        it = iter(clip_generator)
        while True:
            batch = list(itertools.islice(it, self.batch_clips))
            if not batch:
                return
            for spectrogram in generate_features_for_clips(batch, device=self.device):
                yield from split_or_slide(spectrogram, self.step_ms, self.split_spectrogram_duration_s, self.slide_frames)


def write_ragged(out_dir: str, sample_generator, batch_size: int = 100, verbose: bool = False):
    """Store a generator of [T_i, 40] spectrograms as the notebook does (:300-310: ``RaggedMmap.from_generator(out_dir=...,
    sample_generator=..., batch_size=100, verbose=True)``).  With `mmap_ninja` installed this IS that call, so the training
    side (microwakeword/data.py) opens the result unchanged.  Without it (this image has no mmap_ninja and no network) the
    spectrograms go to a documented flat layout -- data.npy = all rows concatenated, starts.npy / ends.npy = row range of
    every sample -- that `read_ragged` opens memory-mapped; the on-disk RaggedMmap layout is deliberately NOT imitated from
    memory, a guess nobody here can check against the library would be worse than an honest different format."""
    try:
        from mmap_ninja.ragged import RaggedMmap
    except ImportError:
        RaggedMmap = None
    if RaggedMmap is not None:
        return RaggedMmap.from_generator(out_dir=out_dir, sample_generator=sample_generator, batch_size=batch_size, verbose=verbose)
    os.makedirs(out_dir, exist_ok=True)
    chunks, starts, ends, pos, dtype, width = [], [], [], 0, None, None
    for sample in sample_generator:
        a = np.ascontiguousarray(sample)
        if a.ndim != 2 or (width is not None and a.shape[1] != width):
            raise ValueError("write_ragged: every sample must be [T, %s]" % (width if width is not None else "F"))
        dtype, width = a.dtype if dtype is None else dtype, a.shape[1]
        chunks.append(a.astype(dtype, copy=False))
        starts.append(pos)
        pos += a.shape[0]
        ends.append(pos)
    data = np.concatenate(chunks, 0) if chunks else np.zeros((0, 40), np.float32)
    np.save(os.path.join(out_dir, "data.npy"), data)
    np.save(os.path.join(out_dir, "starts.npy"), np.asarray(starts, np.int64))
    np.save(os.path.join(out_dir, "ends.npy"), np.asarray(ends, np.int64))
    return read_ragged(out_dir)


class _Ragged:
    def __init__(self, data, starts, ends):
        self.data, self.starts, self.ends = data, starts, ends

    def __len__(self):
        return len(self.starts)

    def __getitem__(self, i):
        if isinstance(i, slice):
            return [self[j] for j in range(*i.indices(len(self)))]
        return self.data[self.starts[i]:self.ends[i]]


def read_ragged(out_dir: str):
    """Open what write_ragged stored: RaggedMmap when mmap_ninja wrote it, else the flat layout (memory-mapped)."""
    if not os.path.exists(os.path.join(out_dir, "data.npy")):
        from mmap_ninja.ragged import RaggedMmap
        return RaggedMmap(out_dir)
    return _Ragged(np.load(os.path.join(out_dir, "data.npy"), mmap_mode="r"), np.load(os.path.join(out_dir, "starts.npy")),
                   np.load(os.path.join(out_dir, "ends.npy")))
