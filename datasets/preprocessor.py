"""Dataset preprocessing on the H100 front-end: wav -> (mu-law / raw audio, mel [frames, 80], linear [frames, n_fft/2+1]) .npy files + the
metadata rows `audio|mel|linear|time_steps|mel_frames|text` (reference datasets/preprocessor.py:12-165). Same step order: load,
optional silence trim, pre-emphasis, separate rescale of the plain and pre-emphasised signals, mu-law + silence clipping when the
WaveNet input is quantised, spectrograms from the PRE-EMPHASISED signal, right zero-padding so that len(audio) == frames * hop.
The reference fans utterances out over processes (the STFT is numpy there); here one process drives the fused STFT / mel kernel."""
import os

import numpy as np

from datasets import audio
from wavenet_vocoder.util import is_mulaw, is_mulaw_quantize, mulaw, mulaw_quantize


def build_from_path(hparams, input_dirs, mel_dir, linear_dir, wav_dir, n_jobs=1, tqdm=lambda x: x):
    """LJSpeech-style folders: `<dir>/metadata.csv` with rows `basename|raw text|normalised text` and `<dir>/wavs/<basename>.wav`."""
    rows = []
    for input_dir in input_dirs:
        with open(os.path.join(input_dir, "metadata.csv"), encoding="utf-8") as f:
            for line in f:
                parts = line.strip().split("|")
                if len(parts) < 2:
                    continue
                # the utterance's basename names its files: audio-<basename>.npy ... (preprocessor.py:33-38); text = third column
                rows.append((parts[0], os.path.join(input_dir, "wavs", "%s.wav" % parts[0]), parts[2] if len(parts) > 2 else parts[-1]))
    out = []
    for basename, wav_path, text in tqdm(rows):
        r = _process_utterance(mel_dir, linear_dir, wav_dir, basename, wav_path, text, hparams)
        if r is not None:
            out.append(r)
    return out


def _process_utterance(mel_dir, linear_dir, wav_dir, index, wav_path, text, hparams):
    try:
        wav = audio.load_wav(wav_path, sr=hparams.sample_rate)
    except FileNotFoundError:
        print("file %s present in csv metadata is not present in wav folder. skipping!" % wav_path)
        return None
    if hparams.trim_silence:
        wav = audio.trim_silence(wav, hparams)
    preem_wav = audio.preemphasis(wav, hparams.preemphasis, hparams.preemphasize)
    if hparams.rescale:
        wav = wav / np.abs(wav).max() * hparams.rescaling_max
        preem_wav = preem_wav / np.abs(preem_wav).max() * hparams.rescaling_max
        if (wav > 1.0).any() or (wav < -1.0).any() or (preem_wav > 1.0).any() or (preem_wav < -1.0).any():
            raise RuntimeError("wav has invalid value: %s" % wav_path)
    wav, preem_wav = wav.astype(np.float32), np.asarray(preem_wav, dtype=np.float32)
    if is_mulaw_quantize(hparams.input_type):
        out = mulaw_quantize(wav, hparams.quantize_channels)
        start, end = audio.start_and_end_indices(out, hparams.silence_threshold)
        wav, preem_wav, out = wav[start:end], preem_wav[start:end], out[start:end]
        constant_values, out_dtype = int(mulaw_quantize(np.zeros(1, dtype=np.float32), hparams.quantize_channels)[0]), np.int16
    elif is_mulaw(hparams.input_type):
        out = mulaw(wav, hparams.quantize_channels)
        constant_values, out_dtype = 0.0, np.float32
    else:
        out, constant_values, out_dtype = wav, 0.0, np.float32
    mel = audio.melspectrogram(preem_wav, hparams).astype(np.float32)             # [num_mels, frames]
    mel_frames = mel.shape[1]
    if mel_frames > hparams.max_mel_frames and hparams.clip_mels_length:
        return None
    linear = audio.linearspectrogram(preem_wav, hparams).astype(np.float32)
    assert linear.shape[1] == mel_frames
    hop = audio.get_hop_size(hparams)
    l_pad, r_pad = audio.librosa_pad_lr(wav, hparams.n_fft, hop, hparams.wavenet_pad_sides)
    out = np.pad(out, (l_pad, r_pad), mode="constant", constant_values=constant_values)
    assert len(out) >= mel_frames * hop
    out = out[:mel_frames * hop]
    time_steps = len(out)
    audio_filename, mel_filename, linear_filename = "audio-%s.npy" % index, "mel-%s.npy" % index, "linear-%s.npy" % index
    np.save(os.path.join(wav_dir, audio_filename), out.astype(out_dtype), allow_pickle=False)
    np.save(os.path.join(mel_dir, mel_filename), mel.T, allow_pickle=False)
    np.save(os.path.join(linear_dir, linear_filename), linear.T, allow_pickle=False)
    return (audio_filename, mel_filename, linear_filename, time_steps, mel_frames, text)
