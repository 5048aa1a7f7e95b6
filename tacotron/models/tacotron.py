"""Python surface of the reference's Tacotron class (tacotron/models/tacotron.py) on top of libt2b200.

As in wavenet_vocoder/models/wavenet.py of this repo, the TF1 graph-building calls execute eagerly:
`initialize(...)` runs the encoder / decoder / postnet (TacoTrainingHelper for training, evaluation and GTA: teacher-forced at
hparams.tacotron_teacher_forcing_ratio, always at ratio 1 for GTA; free-running otherwise), `add_loss()` publishes the four loss terms, `add_optimizer(global_step)` runs BPTT (+ NCCL mean over ranks)
+ clip_by_global_norm + Adam. Attribute names read by tacotron/train.py and tacotron/synthesizer.py are kept
(`tower_mel_outputs`, `tower_alignments`, `tower_stop_token_prediction`, `tower_decoder_output`, `loss`,
`before_loss`, `after_loss`, `stop_token_loss`, `regularization_loss`, `learning_rate`, `gradients`). One process per
GPU replaces the towers. predict_linear (CBHG post-processing net + linear head, tacotron.py:203-219) runs as a second engine chained on
mel_outputs; outputs_per_step > 1 is not implemented (SURVEY.md §8f)."""
import collections

import torch

from t2_import import t2

# Engines are specialised to (B, T_in, T_out) and the reference feeder pads every batch to its own maxima (tacotron/feeder.py:
# 231-256). Padding further is NOT transparent here (batch-norm statistics include the padded frames, modules.py:388), so shapes
# are kept exact and at most `_MAX_ENGINES` engines (with their BPTT workspaces) stay alive, least recently used first out;
# parameters, Adam state and gradients are shared between them.
_MAX_ENGINES = 4


def engine_teacher_forcing_ratio(hparams, gta):
    """Teacher-forcing ratio of the engine behind a teacher-forced graph (helpers.py:86-108): GTA always feeds the targets; training
    and evaluation use hparams.tacotron_teacher_forcing_ratio ('constant' mode; tacotron_natural_eval stays rejected by make_config)."""
    return 1.0 if gta else float(hparams.tacotron_teacher_forcing_ratio)


class Tacotron(object):
    def __init__(self, hparams):
        self._hparams = hparams
        self._engines = collections.OrderedDict()
        self._pending = None

    def _engine(self, B, T_in, T_out, teacher_forcing_ratio=1.0):
        key = (B, T_in, T_out, float(teacher_forcing_ratio))
        if key in self._engines:
            self._engines.move_to_end(key)
            return self._engines[key]
        donor = next(reversed(self._engines.values())) if self._engines else None
        while len(self._engines) >= _MAX_ENGINES:                      # evict BEFORE allocating the new workspace
            _, old = self._engines.popitem(last=False)
            old.workspace = old.packed = None
        eng = t2.tacotron.Tacotron(self._hparams, B, T_in, T_out, teacher_forcing_ratio=teacher_forcing_ratio)
        if donor is not None:
            eng.params, eng.m, eng.v, eng.grads, eng.global_step = donor.params, donor.m, donor.v, donor.grads, donor.global_step
        elif self._pending is not None:
            eng.load_params(self._pending)
            self._pending = None
        else:
            eng.init_variables()
        self._engines[key] = eng
        return eng

    def load_variables(self, name_to_tensor):
        if self._engines:
            next(iter(self._engines.values())).load_params(name_to_tensor)
            for e in self._engines.values():
                e._dirty = True
        else:
            self._pending = name_to_tensor

    def initialize(self, inputs, input_lengths, mel_targets=None, stop_token_targets=None, linear_targets=None, targets_lengths=None,
                   gta=False, global_step=None, is_training=False, is_evaluating=False, split_infos=None):
        """tacotron.py:28-29. inputs int [B, T_in] (0-padded ids), input_lengths [B], mel_targets [B, T_out, num_mels],
        stop_token_targets [B, T_out]. Same argument validation as the reference (tacotron.py:41-54)."""
        hp = self._hparams
        if mel_targets is None and stop_token_targets is not None:
            raise ValueError("no multi targets were provided but token_targets were given")
        if mel_targets is not None and stop_token_targets is None and not gta:
            raise ValueError("Mel targets are provided without corresponding token_targets")
        if not gta and hp.predict_linear and linear_targets is None and is_training:
            raise ValueError("Model is set to use post processing to predict linear spectrograms in training but no linear targets given!")
        if gta and linear_targets is not None:
            raise ValueError("Linear spectrogram prediction is not supported in GTA mode!")
        if is_training and hp.mask_decoder and targets_lengths is None:
            raise RuntimeError("Model set to mask paddings but no targets lengths provided for the mask!")
        if is_training and is_evaluating:
            raise RuntimeError("Model can not be in training and evaluation modes at the same time!")
        if hp.outputs_per_step != 1:
            raise NotImplementedError("outputs_per_step > 1 is out of scope (SURVEY.md §8)")
        post_condition = hp.predict_linear and not gta                 # tacotron.py:109
        self.is_training, self.is_evaluating, self.gta = is_training, is_evaluating, gta
        B, T_in = inputs.shape
        ids, lens = inputs.int().contiguous(), input_lengths.int().contiguous()
        if is_training or is_evaluating or gta:                     # TacoTrainingHelper
            T_out = mel_targets.shape[1]
            eng = self._engine(B, T_in, T_out, engine_teacher_forcing_ratio(hp, gta))
            if global_step is not None:
                eng.global_step = int(global_step)
            stop = stop_token_targets if stop_token_targets is not None else torch.zeros(B, T_out, device=inputs.device)
            eng.step_dev.add_(1)
            lin_t = linear_targets.float().contiguous() if (post_condition and linear_targets is not None) else None
            if post_condition and lin_t is None:                     # evaluation without linear targets: run the head without a loss
                is_lin_train = False
            else:
                is_lin_train = is_training
            eng.forward(ids, lens, mel_targets.float().contiguous(), stop.float().contiguous(), training=is_training and (is_lin_train or not post_condition),
                        targets_lengths=targets_lengths.int().contiguous() if (hp.mask_decoder and targets_lengths is not None) else None,
                        linear_targets=lin_t)
            if post_condition:
                self.tower_linear_outputs = [eng.linear_outputs()]
            M = hp.num_mels
            self.tower_decoder_output = [eng.workspace_tensor("decoder_output", (B, T_out, M))]
            self.tower_mel_outputs = [eng.workspace_tensor("mel_outputs", (B, T_out, M))]
            self.tower_alignments = [eng.workspace_tensor("alignments", (T_out, B, T_in)).permute(1, 2, 0)]  # [B, T_in, T_out] (tacotron.py:222)
            logits = eng.workspace_tensor("stop_logits", (B, T_out))
            self.tower_stop_token_prediction = [logits if (is_training or is_evaluating) else torch.sigmoid(logits)]
        else:                                                       # TacoTestHelper (free running)
            max_iters = min(int(hp.max_iters), int(getattr(hp, "synthesis_max_frames", 2000)))
            eng = self._engine(B, T_in, max_iters)
            out = eng.synthesize(ids, lens)
            self.tower_decoder_output = [out["decoder_output"]]
            self.tower_mel_outputs = [out["mel_outputs"]]
            self.tower_alignments = [out["alignments"].transpose(1, 2)]
            self.tower_stop_token_prediction = [out["stop_token_prediction"]]
            if post_condition:
                self.tower_linear_outputs = [eng.linear_from_mel(out["mel_outputs"])]
        self._eng = eng
        self.tower_linear_targets = [linear_targets]
        self.tower_inputs, self.tower_input_lengths = [inputs], [input_lengths]
        self.tower_mel_targets, self.tower_targets_lengths = [mel_targets], [targets_lengths]
        self.tower_stop_token_targets = [stop_token_targets]
        self.all_vars = eng.params
        return self

    def add_loss(self):
        """tacotron.py:273-369: MSE before + MSE after + stop-token CE (masked variants when hparams.mask_decoder) + L2 regulariser."""
        b = self._eng.loss_buf
        self.tower_before_loss, self.tower_after_loss = [b[0]], [b[1]]
        self.tower_stop_token_loss, self.tower_regularization_loss = [b[2]], [b[3]]
        self.tower_linear_loss = [torch.zeros((), device=b.device)]
        reg = b[3]
        if self._eng.cbhg is not None:                               # tacotron.py:323-345: linear L1 + the CBHG kernels in the regulariser
            self.tower_linear_loss = [self._eng.cb_loss[0]]
            reg = b[3] + self._eng.cb_loss[1]
            self.tower_regularization_loss = [reg]
        self.before_loss, self.after_loss, self.stop_token_loss, self.regularization_loss = b[0], b[1], b[2], reg
        self.linear_loss = self.tower_linear_loss[0]
        self.tower_loss = [b[0] + b[1] + b[2] + reg + self.linear_loss]
        self.loss = self.tower_loss[0]
        return self.loss

    def add_optimizer(self, global_step=None):
        """tacotron.py:371-437: gradients -> mean over ranks -> clip_by_global_norm(1.) -> Adam with the decayed LR."""
        import torch.distributed as dist
        eng = self._eng
        if global_step is not None:
            eng.global_step = int(global_step)
        eng.backward()
        world = dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1
        if world > 1:
            dist.all_reduce(eng.grads, op=dist.ReduceOp.SUM)
        self.learning_rate = eng.optimizer_step(grad_scale=1.0 / world)
        for other in self._engines.values():
            other.global_step, other.m, other.v, other.grads, other._dirty = eng.global_step, eng.m, eng.v, eng.grads, True
        self.gradients = eng.grads
        self.optimize = None
        return self.learning_rate
