"""WaveNet feeder: reads `tacotron_output/gta/map.txt` (rows `audio|mel|gta_mel|speaker_id|text`, tacotron/synthesize.py) or the
preprocessor's `train.txt`, loads audio + conditioning mels and produces hop-aligned, padded batches on a background thread.

Semantics kept from the reference's wavenet_vocoder/feeder.py: deterministic split (`wavenet_data_random_state`, :44-62); crops
of at most max_time_steps (rounded DOWN to a multiple of hop_size) starting at a random frame (:368-387); audio length ==
frames * hop asserted (:400-401); conditioning mels clipped to the Tacotron output range, padded with its minimum and mapped to
[0, 1] (:319-340); inputs padded with zeros. What differs by design: mu-law inputs stay INDICES ([B, T] int32, the one-hot float
[B, 256, T] of :295-306 is never materialised: the first 1x1 convolution is a row gather on the H100 path); tensors are pinned
torch tensors; T is additionally right-padded to a whole hop multiple per batch (it already is, by construction)."""
import os
import queue
import threading

import numpy as np
import torch

from datasets import audio
from wavenet_vocoder.util import is_mulaw_quantize

_batches_per_group = 32


def _round_down(x, multiple):
    return x - x % multiple


def _ensure_divisible(length, divisible_by=256, lower=True):
    if length % divisible_by == 0:
        return length
    return length - length % divisible_by if lower else length + (divisible_by - length % divisible_by)


def _interp(feats, in_range):
    return (feats - in_range[0]) / (in_range[1] - in_range[0])


class Feeder(object):
    def __init__(self, metadata_filename, base_dir, hparams, rank=0, world_size=1, seed=None, prefetch=8):
        self._hparams = hparams
        self._base_dir = base_dir
        with open(metadata_filename, "r", encoding="utf-8") as f:
            self._metadata = [line.strip().split("|") for line in f if line.strip()]
        from sklearn.model_selection import train_test_split
        bs = hparams.wavenet_batch_size
        test_size = hparams.wavenet_test_size if hparams.wavenet_test_size is not None else hparams.wavenet_test_batches * bs
        test_size = int(test_size) if test_size >= 1 else float(test_size)     # sklearn: an int counts examples, a float is a fraction
        idx = np.arange(len(self._metadata))
        train_idx, test_idx = train_test_split(idx, test_size=test_size, random_state=hparams.wavenet_data_random_state)
        keep = _round_down(len(test_idx), bs)
        train_idx = np.concatenate([train_idx, test_idx[keep:]])
        test_idx = test_idx[:keep]
        self._train_meta = [self._metadata[i] for i in train_idx]
        self._test_meta = [self._metadata[i] for i in test_idx]
        self.test_steps = len(self._test_meta) // bs
        self.local_condition = hparams.cin_channels > 0
        self._rank, self._world = rank, world_size
        self._rng = np.random.RandomState(hparams.wavenet_random_seed if seed is None else seed)
        self._train_offset = 0
        self._queue = queue.Queue(maxsize=prefetch)
        self._stop = threading.Event()
        self._thread = None

    def _load(self, meta):
        mel_file = meta[2] if self._hparams.train_with_GTA else meta[1]
        if self._hparams.train_with_GTA and "linear" in mel_file:
            raise RuntimeError("Linear spectrogram files selected instead of GTA mels, did you specify the wrong metadata?")
        x = np.load(os.path.join(self._base_dir, meta[0]))
        c = np.load(os.path.join(self._base_dir, mel_file)) if self.local_condition else None
        if self._global_condition():      # speaker id column (feeder.py:184-189)
            g = meta[3]
            if g == "<no_g>":
                raise RuntimeError("Please redo the wavenet preprocessing (or GTA synthesis) to assign global condition features!")
            return x, c, int(g), len(x)
        return x, c, len(x)

    def _global_condition(self):
        return (getattr(self._hparams, "gin_channels", None) or 0) > 0

    def _next_example(self):
        if self._train_offset >= len(self._train_meta):
            self._train_offset = 0
            self._rng.shuffle(self._train_meta)
        meta = self._train_meta[self._train_offset]
        self._train_offset += 1
        return self._load(meta)

    def _limit_time(self):
        hp = self._hparams
        if hp.max_time_sec is not None:
            return int(hp.max_time_sec * hp.sample_rate)
        return hp.max_time_steps

    def _crop(self, x, c):
        hop = audio.get_hop_size(self._hparams)
        assert len(x) % len(c) == 0 and len(x) // len(c) == hop, "audio / mel lengths are not hop-aligned"
        limit = self._limit_time()
        if limit is not None and len(x) > limit:
            frames = _ensure_divisible(limit, hop, True) // hop
            start = self._rng.randint(0, len(c) - frames)
            x, c = x[start * hop:(start + frames) * hop], c[start:start + frames]
        return x, c

    def prepare_batch(self, batch):
        hp = self._hparams
        items = [self._crop(e[0], e[1]) for e in batch]     # examples are (x, c, len), or (x, c, speaker id, len) with gin
        lengths = np.asarray([len(x) for x, _ in items], dtype=np.int32)
        T = int(lengths.max())
        quant = is_mulaw_quantize(hp.input_type)
        dt = np.int32 if quant else np.float32
        x = np.stack([np.pad(a.astype(dt), (0, T - len(a))) for a, _ in items])
        lo, hi = (-hp.max_abs_value, hp.max_abs_value) if hp.symmetric_mels else (0.0, hp.max_abs_value)
        cs = [np.clip(c, lo, hi) if hp.clip_for_wavenet else c for _, c in items]
        Tc = max(len(c) for c in cs)
        c = np.stack([np.pad(a, [(0, Tc - len(a)), (0, 0)], mode="constant", constant_values=lo) for a in cs]).astype(np.float32)
        c = np.transpose(c, (0, 2, 1))
        if hp.normalize_for_wavenet:
            c = _interp(c, (lo, hi)).astype(np.float32)
        # inputs == targets (the loss shifts by one sample, wavenet.py:488); y keeps the reference's trailing axis
        out = {"inputs": x, "targets": x[:, :, None], "input_lengths": lengths, "local_condition_features": np.ascontiguousarray(c)}
        if self._global_condition():
            out["global_condition_features"] = np.asarray([[e[2]] for e in batch], dtype=np.int32)   # [B, 1] (feeder.py:94-95)
        return out

    def train_group(self):
        n = self._hparams.wavenet_batch_size
        examples = [self._next_example() for _ in range(n * _batches_per_group)]
        examples.sort(key=lambda e: e[-1])
        batches = [examples[i:i + n] for i in range(0, len(examples), n)]
        self._rng.shuffle(batches)
        return [self.prepare_batch(b) for b in batches[self._rank::self._world]]

    def test_batches(self):
        n = self._hparams.wavenet_batch_size
        examples = sorted((self._load(m) for m in self._test_meta), key=lambda e: e[-1])
        return [self.prepare_batch(examples[i:i + n]) for i in range(0, len(examples), n)]

    @staticmethod
    def to_tensors(batch, pin=True):
        out = {k: torch.from_numpy(v) for k, v in batch.items()}
        if pin and torch.cuda.is_available():
            out = {k: v.pin_memory() for k, v in out.items()}
        return out

    def _run(self):
        while not self._stop.is_set():
            for b in self.train_group():
                t = self.to_tensors(b)
                while not self._stop.is_set():
                    try:
                        self._queue.put(t, timeout=0.2)
                        break
                    except queue.Full:
                        continue
                if self._stop.is_set():
                    return

    def start(self):
        self._thread = threading.Thread(target=self._run, name="wavenet-feeder", daemon=True)
        self._thread.start()
        return self

    def next_batch(self, timeout=600):
        if self._thread is None:
            self.start()
        return self._queue.get(timeout=timeout)

    def stop(self):
        self._stop.set()
        if self._thread is not None:
            self._thread.join(timeout=5)
