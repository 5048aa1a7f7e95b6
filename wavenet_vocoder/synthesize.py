"""WaveNet synthesis driver (reference wavenet_vocoder/synthesize.py:12-80): every mel-*.npy of --mels_dir (or the map.txt of a
Tacotron eval run when --model Tacotron-2) -> <output>/wavs/wavenet-audio-*.wav + map.txt."""
import os

import numpy as np

import t2_checkpoint
from infolog import log
from wavenet_vocoder.synthesizer import Synthesizer


def run_synthesis(args, checkpoint_path, output_dir, hparams):
    wav_dir, log_dir = os.path.join(output_dir, "wavs"), os.path.join(output_dir, "plots")
    os.makedirs(wav_dir, exist_ok=True)
    os.makedirs(log_dir, exist_ok=True)
    synth = Synthesizer()
    synth.load(checkpoint_path, hparams)
    if args.model == "Tacotron-2":
        with open(os.path.join(args.mels_dir, "map.txt"), encoding="utf-8") as f:
            rows = [line.strip().split("|") for line in f if line.strip()]
        texts, mel_files = [r[0] for r in rows], [r[1] for r in rows]
        speaker_ids = [r[2] if len(r) > 2 else "<no_g>" for r in rows]            # speaker column (wavenet_vocoder/synthesize.py:26-30)
        speaker_ids = None if all(s == "<no_g>" for s in speaker_ids) else speaker_ids
    else:
        mel_files = sorted(os.path.join(args.mels_dir, f) for f in os.listdir(args.mels_dir) if f.endswith(".npy"))
        texts = None
        sid = getattr(args, "speaker_id", None)                                      # --speaker_id "0,3,1,..." (:33-36)
        speaker_ids = None if sid is None else sid.replace(" ", "").split(",")
        if speaker_ids is not None and len(speaker_ids) != len(mel_files):
            raise ValueError("--speaker_id has %d ids for %d mel files" % (len(speaker_ids), len(mel_files)))
    log("Starting synthesis! (this will take a while..)")
    n = hparams.wavenet_synthesis_batch_size
    with open(os.path.join(wav_dir, "map.txt"), "w", encoding="utf-8") as f:
        for i in range(0, len(mel_files), n):
            batch = mel_files[i:i + n]
            mels = [np.load(m) for m in batch]
            basenames = [os.path.basename(m).replace(".npy", "") for m in batch]
            audio_files = synth.synthesize(mels, None if speaker_ids is None else speaker_ids[i:i + n], basenames, wav_dir, log_dir)
            for j, mel_file in enumerate(batch):
                f.write(("%s|%s\n" % (mel_file, audio_files[j])) if texts is None else ("%s|%s|%s\n" % (texts[i + j], mel_file, audio_files[j])))
    log("synthesized audio waveforms at %s" % wav_dir)
    return wav_dir


def wavenet_synthesize(args, hparams, checkpoint):
    output_dir = "wavenet_" + args.output_dir
    path = t2_checkpoint.latest(checkpoint)
    if path is None:
        raise RuntimeError("Failed to load checkpoint at %s" % checkpoint)
    log("loaded model at %s" % path)
    return run_synthesis(args, path, output_dir, hparams)
