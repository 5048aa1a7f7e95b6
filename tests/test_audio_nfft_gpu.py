"""GPU audio front-end and Griffin-Lim at every supported n_fft (512, 1024, 2048, 4096) against the numpy oracle, at the
(sample rate, n_fft, hop, window) points of an 8 to 48 kHz corpus, plus preprocess -> Tacotron (predict_linear) -> synthesis
previews on 16 and 48 kHz toy corpora.

Tolerances as in test_audio_gpu.py: spectrograms within 1e-3 absolute in the normalised [-4, 4] domain; Griffin-Lim waveforms
from the same injected phases within 2e-4 (0 rounds) and 5e-3 (3 rounds) of the signal's peak."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from audio_nfft_points import POINTS, hp_for, point_id
from oracle import audio as oa
from t2_import import t2

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WIN_NONE = (16000, 1024, 200, None)      # win_size=None: the window spans the whole n_fft frame


def _oracle_hp(hp):
    ohp = hp.copy()
    if ohp.win_size is None:
        ohp.set_hparam("win_size", hp.n_fft)
    return ohp


def _wav(seed, n, sr):
    """chirp from 100 Hz to 0.4 sr plus noise, peak 0.999"""
    rng = np.random.default_rng(seed)
    t = np.arange(n) / float(sr)
    w = 0.5 * np.sin(2 * np.pi * (100 + 0.2 * sr * t / t[-1]) * t) + rng.normal(0, 0.05, n)
    return (w / np.abs(w).max() * 0.999).astype(np.float32)


def _err(a, b):
    return float(np.abs(np.asarray(a, dtype=np.float64) - b).max())


@pytest.mark.parametrize("point", POINTS + [WIN_NONE], ids=point_id)
def test_spectrograms_match_oracle(point):
    hp = hp_for(*point)
    ohp = _oracle_hp(hp)
    sr, n_fft, hop = point[0], point[1], point[2]
    nm, bins = hp.num_mels, n_fft // 2 + 1
    fe = t2.audio.MelFrontEnd(hp)
    n_long = int(0.73 * sr) + 7                 # not a whole number of hops at any point
    n_short = n_fft * 3 // 5                    # a clip shorter than one frame
    for B, n in ((3, n_long), (1, n_short)):
        wavs = np.stack([oa.preemphasis(_wav(s, n, sr), 0.97).astype(np.float32) for s in range(B)])
        x = torch.from_numpy(wavs).cuda()
        mel, lin = fe(x, linear=True)
        mel_t, lin_t = fe(x, time_major=False, linear=True)
        frames = n // hop + 1
        assert mel.shape == (B, frames, nm) and lin.shape == (B, frames, bins)
        assert mel_t.shape == (B, nm, frames) and lin_t.shape == (B, bins, frames)
        for i in range(B):
            ref, lref = oa.melspectrogram(wavs[i], ohp), oa.linearspectrogram(wavs[i], ohp)
            errs = (_err(mel[i].cpu().numpy().T, ref), _err(mel_t[i].cpu().numpy(), ref),
                    _err(lin[i].cpu().numpy().T, lref), _err(lin_t[i].cpu().numpy(), lref))
            assert max(errs) < 1e-3, "B=%d n=%d item %d: mel / mel_t / lin / lin_t max abs err %s" % (B, n, i, errs)
    # pre-emphasis and gain fused into the STFT load
    w = _wav(7, n_long, sr)
    pre = oa.preemphasis(w, 0.97)
    gain = 0.999 / np.abs(pre).max()
    out = fe(torch.from_numpy(w[None]).cuda(), preemphasis=0.97, gain=float(gain))[0].cpu().numpy().T
    assert _err(out, oa.melspectrogram(pre * gain, ohp)) < 1e-3
    # silence lands on the floor, clipped to -max_abs_value
    m, l = fe(torch.zeros(2, n_long, device="cuda"), linear=True)
    assert torch.all(m == -hp.max_abs_value) and torch.all(l == -hp.max_abs_value)


@pytest.mark.parametrize("point", POINTS + [WIN_NONE], ids=point_id)
def test_griffin_lim_matches_oracle_with_injected_phases(point):
    hp = hp_for(*point)
    ohp = _oracle_hp(hp)
    hop, frames = point[2], 24
    rng = np.random.default_rng(point[1])
    n = hop * (frames - 1)
    y0 = (0.4 * np.sin(np.arange(n) * 0.05) + 0.05 * rng.standard_normal(n)).astype(np.float32)
    S = np.abs(oa.stft(y0, ohp)).astype(np.float64)                 # [bins, frames]
    assert S.shape == (point[1] // 2 + 1, frames)
    ang = np.exp(2j * np.pi * rng.random(S.shape))
    fe = t2.audio.MelFrontEnd(hp)
    mag = torch.from_numpy(np.ascontiguousarray(S.T, dtype=np.float32))[None].cuda()
    for iters, tol in ((0, 2e-4), (3, 5e-3)):
        ref = oa.griffin_lim(S, ohp, ang, iters=iters)
        ph = torch.from_numpy(np.stack([ang.real.T, ang.imag.T], axis=-1).astype(np.float32))[None].contiguous().cuda()
        wav = fe.griffin_lim(mag, iters, phase=ph)[0].cpu().numpy()
        assert wav.shape == ref.shape == (n,)
        rel = np.abs(wav - ref).max() / np.abs(ref).max()
        assert rel < tol, "iters %d: max err / max |y| = %.3g" % (iters, rel)
    # the self-seeded path converges
    e = [np.abs(np.abs(oa.stft(fe.griffin_lim(mag, it, seed=7)[0].cpu().numpy(), ohp)) - S).mean() for it in (0, 30)]
    assert e[1] < 0.5 * e[0], e


# ---- preprocess.py -> Tacotron with the linear head -> synthesis previews ----------------------------------------------------------
TOY = ("enc_conv_channels=256,embedding_dim=256,encoder_lstm_units=128,decoder_lstm_units=256,postnet_channels=256,"
       "prenet_layers=[128,128],attention_dim=128,tacotron_batch_size=4,tacotron_test_size=4,tacotron_test_batches=None,max_iters=60,"
       "tacotron_synthesis_batch_size=4,input_type=raw,trim_silence=False")


def _run(args, cwd):
    env = dict(os.environ, PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable] + args, cwd=cwd, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, "%s\nSTDOUT:\n%s\nSTDERR:\n%s" % (" ".join(args), r.stdout[-3000:], r.stderr[-3000:])
    return r.stdout


@pytest.mark.parametrize("point", [POINTS[1], POINTS[4]], ids=point_id)
def test_corpus_preprocess_train_synthesize(point, tmp_path):
    from scipy.io import wavfile
    from datasets import audio
    from tacotron.models import create_model
    sr, n_fft, hop, win = point
    bins = n_fft // 2 + 1
    hp_str = TOY + ",sample_rate=%d,n_fft=%d,hop_size=%d,win_size=%d,num_freq=%d,fmax=%d" % (sr, n_fft, hop, win, bins, min(7600, sr // 2))
    hp = hp_for(*point)
    hp.parse(TOY)
    base = str(tmp_path)
    ds = os.path.join(base, "LJSpeech-1.1")
    os.makedirs(os.path.join(ds, "wavs"))
    rng = np.random.default_rng(sr)
    rows = []
    for i in range(6):
        n = int(rng.integers(int(0.4 * sr), int(0.6 * sr)))
        t = np.arange(n) / float(sr)
        w = 0.4 * np.sin(2 * np.pi * (220 + 30 * i) * t * (1 + 0.3 * t)) + 0.02 * rng.standard_normal(n)
        wavfile.write(os.path.join(ds, "wavs", "LJ%03d.wav" % i), sr, (w * 32767).astype(np.int16))
        rows.append("LJ%03d|Sentence %d.|sentence number %d of the toy corpus." % (i, i, i))
    open(os.path.join(ds, "metadata.csv"), "w").write("\n".join(rows) + "\n")

    out = _run([os.path.join(ROOT, "preprocess.py"), "--base_dir", base, "--hparams", hp_str], base)
    assert "Write 6 utterances" in out
    td = os.path.join(base, "training_data")
    meta = [l.strip().split("|") for l in open(os.path.join(td, "train.txt"))]
    assert len(meta) == 6
    mels, lins = [], []
    for m in meta:
        mel, lin = np.load(os.path.join(td, "mels", m[1])), np.load(os.path.join(td, "linear", m[2]))
        frames = int(m[4])
        assert mel.shape == (frames, 80) and lin.shape == (frames, bins) and int(m[3]) == frames * hop
        # the reference's steps on the host: load, pre-emphasis, rescale, float32, then the numpy STFT
        wav = audio.load_wav(os.path.join(ds, "wavs", m[0][len("audio-"):-len(".npy")] + ".wav"), sr)
        pre = oa.preemphasis(wav, hp.preemphasis)
        pre = (pre / np.abs(pre).max() * hp.rescaling_max).astype(np.float32)
        assert _err(mel.T, oa.melspectrogram(pre, hp)) < 1e-3 and _err(lin.T, oa.linearspectrogram(pre, hp)) < 1e-3
        mels.append(mel)
        lins.append(lin)

    # one drop-in training step of the mel predictor + CBHG linear head on these targets
    assert hp.predict_linear and hp.num_freq == bins
    T_out = min(x.shape[0] for x in mels[:4])
    mel_t = torch.from_numpy(np.stack([x[:T_out] for x in mels[:4]])).cuda()
    lin_t = torch.from_numpy(np.stack([x[:T_out] for x in lins[:4]])).cuda()
    stop = torch.zeros(4, T_out, device="cuda")
    stop[:, -1] = 1
    g = torch.Generator().manual_seed(0)
    ids = torch.randint(2, 66, (4, 20), generator=g).cuda()
    lens = torch.tensor([20, 18, 15, 11]).cuda()
    model = create_model("Tacotron", hp)
    model.initialize(ids, lens, mel_t, stop, linear_targets=lin_t, global_step=0, is_training=True)
    loss = float(model.add_loss())
    model.add_optimizer(0)
    assert np.isfinite(loss) and loss > 0
    assert model.tower_linear_outputs[0].shape == (4, T_out, bins) and torch.isfinite(model.tower_linear_outputs[0]).all()

    # Griffin-Lim inversions of the preprocessed spectrograms
    for spec, inv in ((lins[0], audio.inv_linear_spectrogram), (mels[0], audio.inv_mel_spectrogram)):
        y = inv(spec.T, hp)
        assert y.shape == (hop * (spec.shape[0] - 1),) and np.isfinite(y).all()

    # the command-line workflow: train.py --model Tacotron, then synthesize.py --mode eval with its Griffin-Lim preview
    common = ["--base_dir", base, "--hparams", hp_str, "--name", "nfft", "--input_dir", td, "--checkpoint_interval", "2", "--eval_interval", "2"]
    _run([os.path.join(ROOT, "train.py"), "--model", "Tacotron", "--tacotron_train_steps", "2"] + common, base)
    assert os.path.isfile(os.path.join(base, "logs-nfft", "taco_pretrained", "tacotron_model.ckpt-2.npz"))
    txt = os.path.join(base, "sentences.txt")
    open(txt, "w").write("A short test.\n")
    _run([os.path.join(ROOT, "synthesize.py"), "--model", "Tacotron", "--mode", "eval", "--name", "nfft", "--hparams", hp_str, "--text_list", txt], base)
    ev = os.path.join(base, "tacotron_output", "eval")
    lin = np.load(os.path.join(ev, "linear-batch_0_sentence_0.npy"))
    mel = np.load(os.path.join(ev, "mel-batch_0_sentence_0.npy"))
    assert lin.shape == (mel.shape[0], bins) and np.isfinite(lin).all()
    preview = os.path.join(base, "tacotron_output", "logs-eval", "wavs", "wav-batch_0_sentence_0-linear.wav")
    if mel.shape[0] >= 2:       # previews need two frames; the length is the index of the first fired stop token
        rate, data = wavfile.read(preview)
        assert rate == sr and len(data) == hop * (mel.shape[0] - 1)
