"""WaveNet training loop (reference wavenet_vocoder/train.py:222-330): feeder thread -> create_model('WaveNet') ->
initialize / add_loss / add_optimizer per batch, periodic evaluation, checkpoints under
<log_dir>/wave_pretrained/wavenet_model.ckpt-<step>.npz. One process per GPU (torchrun) replaces the towers."""
import os
import time

import numpy as np
import torch

import infolog
import t2_checkpoint
from tacotron.train import ValueWindow, _cuda, _dist
from wavenet_vocoder.feeder import Feeder
from wavenet_vocoder.models import create_model

log = infolog.log


def _run_model(model, b, training):
    x = b["inputs"]
    y = b["targets"]
    g = b.get("global_condition_features")      # speaker ids [B, 1] when gin_channels > 0
    if training:
        model.initialize(y, b["local_condition_features"], g, b["input_lengths"], x=x)
    else:
        model.initialize(y, b["local_condition_features"], g, b["input_lengths"])
    return model.add_loss()


def train(log_dir, args, hparams, input_path):
    rank, world = _dist()
    save_dir = os.path.join(log_dir, "wave_pretrained")
    eval_dir = os.path.join(log_dir, "eval-dir")
    os.makedirs(save_dir, exist_ok=True)
    os.makedirs(eval_dir, exist_ok=True)
    input_path = os.path.join(args.base_dir, input_path)
    log("Checkpoint_path: %s" % os.path.join(save_dir, "wavenet_model.ckpt"))
    log("Loading training data from: %s" % input_path)
    log("Using model: %s" % args.model)
    torch.manual_seed(hparams.wavenet_random_seed)
    feeder = Feeder(input_path, args.base_dir, hparams, rank=rank, world_size=world)
    model = create_model("WaveNet", hparams)
    step = 0
    if args.restore:
        path = t2_checkpoint.latest(save_dir)
        if path:
            log("Loading checkpoint %s" % path)
            variables, state = t2_checkpoint.load(path)
            model.load_variables(variables)
            model._restore_state = state
            step = state["global_step"]
        else:
            log("No model to load at %s" % save_dir)
    else:
        log("Starting new training!")
    feeder.start()
    time_window, loss_window = ValueWindow(100), ValueWindow(100)
    log("Wavenet training set to a maximum of %d steps" % args.wavenet_train_steps)
    try:
        while step < args.wavenet_train_steps:
            t0 = time.time()
            b = _cuda(feeder.next_batch())
            loss = _run_model(model, b, True)
            state = getattr(model, "_restore_state", None)
            if state is not None:
                t2_checkpoint.restore_engine(model._eng, model._eng.export_params(), state)
                model._restore_state = None
            model.add_optimizer(step)
            step += 1
            loss = float(loss)
            time_window.append(time.time() - t0)
            loss_window.append(loss)
            log("Step %7d [%.3f sec/step, loss=%.5f, avg_loss=%.5f]" % (step, time_window.average, loss, loss_window.average),
                end="\r" if step % 10 else "\n")
            if np.isnan(loss) or loss > 100.0:
                log("Loss exploded to %.5f at step %d" % (loss, step))
                raise Exception("Loss exploded")
            if step % args.eval_interval == 0 and feeder.test_steps > 0:
                log("\nEvaluating at step %d" % step)
                losses = [float(_run_model(model, _cuda(Feeder.to_tensors(tb)), False)) for tb in feeder.test_batches()]
                log("Eval loss for global step %d: %.3f" % (step, float(np.mean(losses))))
            if (step % args.checkpoint_interval == 0 or step == args.wavenet_train_steps) and rank == 0:
                path = t2_checkpoint.save(save_dir, "wavenet_model.ckpt", model._eng)
                log("\nSaving Model at step %d: %s" % (step, path))
        log("Wavenet training complete after %d global steps" % args.wavenet_train_steps)
        return save_dir
    finally:
        feeder.stop()


def wavenet_train(args, log_dir, hparams, input_path):
    return train(log_dir, args, hparams, input_path)
