"""python synthesize.py --model Tacotron|WaveNet|Tacotron-2 --mode eval|synthesis [--checkpoint pretrained/] [--text_list F] ...
Same flags as the reference's synthesize.py:47-96."""
import argparse
import os
from time import sleep
from warnings import warn

from hparams import hparams as default_hparams
from infolog import log
from tacotron.synthesize import tacotron_synthesize
from wavenet_vocoder.synthesize import wavenet_synthesize


def prepare_run(args):
    modified_hp = default_hparams.copy().parse(args.hparams)
    run_name = args.name or args.tacotron_name or args.model
    taco_checkpoint = os.path.join("logs-" + run_name, "taco_" + args.checkpoint)
    run_name = args.name or args.wavenet_name or args.model
    wave_checkpoint = os.path.join("logs-" + run_name, "wave_" + args.checkpoint)
    return taco_checkpoint, wave_checkpoint, modified_hp


def get_sentences(args):
    if args.text_list != "":
        with open(args.text_list, "rb") as f:
            return [line.decode("utf-8").strip() for line in f if line.strip()]
    from hparams import sentences
    return list(sentences)


def synthesize(args, hparams, taco_checkpoint, wave_checkpoint, sentences):
    log("Running End-to-End TTS Evaluation. Model: %s" % (args.name or args.model))
    log("Synthesizing mel-spectrograms from text..")
    wavenet_in_dir = tacotron_synthesize(args, hparams, taco_checkpoint, sentences)
    sleep(0.5)
    log("Synthesizing audio from mel-spectrograms.. (This may take a while)")
    args.mels_dir = wavenet_in_dir
    wavenet_synthesize(args, hparams, wave_checkpoint)
    log("Tacotron-2 TTS synthesis complete!")


def main():
    accepted_modes = ["eval", "synthesis", "live"]
    parser = argparse.ArgumentParser()
    parser.add_argument("--checkpoint", default="pretrained/", help="Path to model checkpoint")
    parser.add_argument("--hparams", default="", help="Hyperparameter overrides as a comma-separated list of name=value pairs")
    parser.add_argument("--name", help="Name of logging directory if the two models were trained together.")
    parser.add_argument("--tacotron_name", help="Name of logging directory of Tacotron. If trained separately")
    parser.add_argument("--wavenet_name", help="Name of logging directory of WaveNet. If trained separately")
    parser.add_argument("--model", default="Tacotron-2")
    parser.add_argument("--input_dir", default="training_data/", help="folder to contain inputs sentences/targets")
    parser.add_argument("--mels_dir", default="tacotron_output/eval/", help="folder to contain mels to synthesize audio from using the Wavenet")
    parser.add_argument("--output_dir", default="output/", help="folder to contain synthesized mel spectrograms")
    parser.add_argument("--mode", default="eval", help="mode of run: can be one of %s" % accepted_modes)
    parser.add_argument("--GTA", default="True", help="Ground truth aligned synthesis, defaults to True, only considered in synthesis mode")
    parser.add_argument("--text_list", default="", help="Text file contains list of texts to be synthesized. Valid if mode=eval")
    parser.add_argument("--speaker_id", default=None,
                        help="Comma-separated speaker ids, one per mel file of --mels_dir (WaveNet with gin_channels > 0).")
    args = parser.parse_args()
    accepted_models = ["Tacotron", "WaveNet", "Tacotron-2"]
    if args.model not in accepted_models:
        raise ValueError("please enter a valid model to synthesize with: %s" % accepted_models)
    if args.mode not in accepted_modes:
        raise ValueError("accepted modes are: %s, found %s" % (accepted_modes, args.mode))
    if args.mode == "live" and args.model == "Wavenet":
        raise RuntimeError("Wavenet vocoder cannot be tested live due to its slow generation. Live only works with Tacotron!")
    if args.GTA not in ("True", "False"):
        raise ValueError("GTA option must be either True or False")
    if args.model == "Tacotron-2":
        if args.mode == "live":
            warn("Requested a live evaluation with Tacotron-2, Wavenet will not be used!")
        if args.mode == "synthesis":
            raise ValueError("I don't recommend running WaveNet on entire dataset.. The world might end before the synthesis :) (only eval allowed)")
    taco_checkpoint, wave_checkpoint, hparams = prepare_run(args)
    sentences = get_sentences(args)
    if args.model == "Tacotron":
        tacotron_synthesize(args, hparams, taco_checkpoint, sentences)
    elif args.model == "WaveNet":
        wavenet_synthesize(args, hparams, wave_checkpoint)
    else:
        synthesize(args, hparams, taco_checkpoint, wave_checkpoint, sentences)


if __name__ == "__main__":
    main()
