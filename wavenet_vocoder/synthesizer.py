"""WaveNet Synthesizer (reference wavenet_vocoder/synthesizer.py:14-130): mels [frames, num_mels] -> waveforms through the
autoregressive CUDA generator; conditioning is clipped / padded / mapped to [0, 1] exactly as in training (:59-70)."""
import os

import numpy as np
import torch

import t2_checkpoint
from datasets.audio import get_hop_size, melspectrogram, save_wavenet_wav
from wavenet_vocoder import util
from wavenet_vocoder.models import create_model


class Synthesizer(object):
    def load(self, checkpoint_path, hparams, model_name="WaveNet"):
        self._hparams = hparams
        self.model = create_model(model_name, hparams)
        variables, state = t2_checkpoint.load(checkpoint_path)
        if state["ema"]:            # the reference restores the EMA shadows for synthesis (wavenet_vocoder/synthesizer.py:33-36, train.py:75-83)
            variables = dict(variables, **state["ema"])
        self.model.load_variables(variables)

    def synthesize(self, mel_spectrograms, speaker_ids, basenames, out_dir, log_dir):
        hp = self._hparams
        hop = get_hop_size(hp)
        audio_lengths = [len(x) * hop for x in mel_spectrograms]
        maxlen = max(len(x) for x in mel_spectrograms)
        lo, hi = (-hp.max_abs_value, hp.max_abs_value) if hp.symmetric_mels else (0.0, hp.max_abs_value)
        if hp.clip_for_wavenet:
            mel_spectrograms = [np.clip(x, lo, hi) for x in mel_spectrograms]
        c = np.stack([np.pad(x, [(0, maxlen - len(x)), (0, 0)], mode="constant", constant_values=lo) for x in mel_spectrograms]).astype(np.float32)
        if hp.normalize_for_wavenet:
            c = ((c - lo) / (hi - lo)).astype(np.float32)
        if maxlen == 0:             # every mel is empty (an untrained Tacotron can fire its stop token on the first frame)
            wavs = np.zeros((len(mel_spectrograms), 0), dtype=np.float32)
        else:
            g = None if speaker_ids is None else torch.tensor([[int(s)] for s in speaker_ids], dtype=torch.int32)   # [batch, 1]
            self.model.initialize(None, torch.from_numpy(c).cuda(), g, None)   # c: [batch, frames, num_mels] (wavenet.py:408-427)
            wavs = self.model.tower_y_hat[0].cpu().numpy()
        names = []
        for w, n, b in zip(wavs, audio_lengths, basenames):
            path = os.path.join(out_dir, "wavenet-audio-%s.wav" % b)
            save_wavenet_wav(w[:n], path, sr=hp.sample_rate, inv_preemphasize=hp.preemphasize, k=hp.preemphasis)
            names.append(path)
        if log_dir is not None:         # wavenet_vocoder/synthesizer.py:116-128: the waveform and its mel next to the conditioning mel
            for w, n, b, m in zip(wavs, audio_lengths, basenames, mel_spectrograms):
                if n < hp.n_fft:
                    continue
                util.waveplot(os.path.join(log_dir, "wavenet-waveplot-%s.png" % b), w[:n], None, hp, title="WaveNet generated Waveform.")
                generated_mel = melspectrogram(np.ascontiguousarray(w[:n], dtype=np.float32), hp).T
                util.plot_spectrogram(generated_mel, os.path.join(log_dir, "wavenet-mel-spectrogram-%s.png" % b),
                                      title="Local Condition vs Reconstructed Audio Mel-Spectrogram analysis", target_spectrogram=m)
        return names
