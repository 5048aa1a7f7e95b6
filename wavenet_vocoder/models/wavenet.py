"""Python surface of the reference's WaveNet class (wavenet_vocoder/models/wavenet.py) on top of libt2b200.

The TF1 original builds graph nodes in `initialize` / `add_loss` / `add_optimizer` and runs them later with
`sess.run([model.loss, model.optimize])` (wavenet_vocoder/train.py:303). There is no graph here, so the same three calls
EXECUTE: `initialize(...)` runs the teacher-forced forward (or the autoregressive synthesis), `add_loss()` publishes
the loss, `add_optimizer(global_step)` runs backward (+ NCCL mean over ranks) + clip + Adam + EMA. A training loop
calls the three per batch; the attribute names the reference's loops read (`loss`, `learning_rate`, `tower_y_hat`,
`tower_upsampled_local_features`, ...) are kept. Tensors are torch CUDA tensors; one process per GPU replaces towers
(`wavenet_num_gpus` is the world size of torch.distributed)."""
import collections

import torch

from datasets.audio import get_hop_size
from t2_import import t2
from wavenet_vocoder.util import is_mulaw, is_mulaw_quantize, is_scalar_input

# Engines are specialised to (B, T): the reference feeders pad every batch to its own maximum, so shapes change from step to
# step. T is therefore rounded up to a multiple of `_BUCKET_FRAMES` hops (right padding cannot influence earlier outputs of a
# causal network and the loss is length-masked), and at most `_MAX_ENGINES` shape-specialised engines (workspaces of 1.6-13 GB
# at the paper widths) stay alive, least recently used first out. Parameters, Adam state, EMA and gradients are shared.
_BUCKET_FRAMES = 8
_MAX_ENGINES = 3


class WaveNet(object):
    def __init__(self, hparams, init=False):
        self._hparams = hparams
        self._init = init               # data-dependent weight-norm init of the reference: weight norm is out of scope (§8)
        self._engines = collections.OrderedDict()
        self._synths = collections.OrderedDict()
        self._state = None               # (params, m, v, ema, global_step) shared between shape-specialised engines
        self.variables = None
        self.ema = None

    # ---- reference helpers -------------------------------------------------------------------------------
    def local_conditioning_enabled(self):
        return self._hparams.cin_channels > 0

    def global_conditioning_enabled(self):
        return self._hparams.gin_channels > 0

    def set_mode(self, is_training):
        self.is_training = is_training

    def _engine(self, B, T):
        key = (B, T)
        if key in self._engines:
            self._engines.move_to_end(key)
            return self._engines[key]
        donor = next(reversed(self._engines.values())) if self._engines else None
        while len(self._engines) >= _MAX_ENGINES:                      # evict BEFORE allocating the new workspace
            _, old = self._engines.popitem(last=False)
            old.workspace = old.packed = None
        eng = t2.wavenet.WaveNet(self._hparams, B, T)
        if donor is not None:
            eng.params, eng.m, eng.v, eng.ema, eng.grads = donor.params, donor.m, donor.v, donor.ema, donor.grads   # shared flat buffers
            eng.global_step = donor.global_step
        else:
            eng.init_variables()
        self._engines[key] = eng
        return eng

    def load_variables(self, name_to_tensor):
        """restore from {TF variable name: array}"""
        for eng in self._engines.values():
            eng.load_params(name_to_tensor)
        self._pending = name_to_tensor

    # ---- graph-building calls of the reference, executed eagerly ----------------------------------------------
    def initialize(self, y, c, g, input_lengths, x=None, synthesis_length=None, test_inputs=None, split_infos=None):
        """wavenet.py:218. Training: x = inputs ([B, T] mu-law indices, one-hot float [B, Q, T], or raw [B, 1, T] / [B, T]),
        y = targets ([B, T] or [B, T, 1]), c = local conditioning [B, cin, Tc], input_lengths [B]. Synthesis (x is None and
        y is None): c + synthesis_length (+ test_inputs for teacher-forced debugging). g: speaker ids [B, 1] or [B] (gin_channels > 0),
        or None for no speaker term."""
        hp = self._hparams
        if g is not None and not self.global_conditioning_enabled():
            raise ValueError("speaker ids given but gin_channels = %r (global conditioning is off)" % hp.gin_channels)
        self.is_training = x is not None
        self.is_evaluating = not self.is_training and y is not None
        scalar = is_scalar_input(hp.input_type)
        if self.is_training or self.is_evaluating:
            tgt = y.squeeze(-1) if y.dim() == 3 else y              # targets [B, T, 1] (feeder.py:308-317) or [B, T]
            if x is None:                                           # evaluation: the targets are also the teacher-forcing inputs
                src = tgt
            elif not scalar and x.dim() == 3:                       # one-hot float [B, Q, T] -> indices (feeder.py:295-306)
                src = x.argmax(dim=1)
            elif scalar and x.dim() == 3:                           # [B, 1, T]
                src = x.squeeze(1)
            else:
                src = x
            xin = src.float().contiguous() if scalar else src.int().contiguous()
            tin = tgt.float().contiguous() if scalar else tgt.int().contiguous()
            B, T = xin.shape
            hop = get_hop_size(hp) if self.local_conditioning_enabled() else 1
            if self.local_conditioning_enabled() and T % hop:
                raise t2.lib.T2Error("audio length %d is not a multiple of hop_size %d (wavenet_vocoder/feeder.py:400-401 guarantees it)" % (T, hop))
            Tb = -(-T // (hop * _BUCKET_FRAMES)) * (hop * _BUCKET_FRAMES)
            if Tb != T:                                                # right-pad to the bucket; lengths keep masking the loss
                xin = torch.nn.functional.pad(xin, (0, Tb - T), value=0.0 if scalar else (hp.quantize_channels - 1) // 2)
                tin = torch.nn.functional.pad(tin, (0, Tb - T), value=0.0 if scalar else (hp.quantize_channels - 1) // 2)
                if c is not None:
                    c = torch.nn.functional.pad(c, (0, Tb // hop - c.shape[-1]))
            self._T_valid, T = T, Tb
            eng = self._engine(B, T)
            if getattr(self, "_pending", None) is not None:
                eng.load_params(self._pending)
                self._pending = None
            self._eng = eng
            ldo = 256 if is_mulaw_quantize(hp.input_type) else 32
            self._logits = torch.empty(B, T, ldo, device=xin.device) if getattr(hp, "keep_logits", False) else None
            eng.training = self.is_training
            if self.global_conditioning_enabled():
                eng.set_speakers(g)
            eng.step_dev.add_(1)
            eng.forward(xin, c.float().contiguous(), tin, input_lengths.int().contiguous(), logits=self._logits,
                        save_for_backward=self.is_training)
            Tv = self._T_valid
            self.tower_y = [tin[:, :Tv]]
            self.tower_input_lengths = [input_lengths]
            self.tower_c = [c]
            self.tower_upsampled_local_features = [eng.workspace_tensor("c_up", (B, T, hp.cin_channels))[:, :Tv]]
            self.tower_y_hat = [self._logits[:, :Tv, :hp.out_channels].transpose(1, 2)] if self._logits is not None else []
            self.variables = eng.params
            self.ema = eng.ema
        else:
            # wavenet.py:408-427: c arrives as [batch, local_condition_time, cin_channels]; the synthesis length is OVERWRITTEN by
            # Tc * hop_size and c is transposed to channels-first
            if c is None:
                raise NotImplementedError("unconditional synthesis (cin_channels < 0) is out of scope (SURVEY.md §8)")
            if c.dim() != 3 or c.shape[-1] != hp.cin_channels:
                raise ValueError("Expected 3 dimension shape [batch_size(1), time_length, %d] for local condition features but found %s"
                                 % (hp.cin_channels, tuple(c.shape)))
            B, Tc = c.shape[0], c.shape[1]
            T = Tc * get_hop_size(hp)
            c = c.transpose(1, 2)
            key = (B, T)
            if key in self._synths:
                self._synths.move_to_end(key)
            else:
                while len(self._synths) >= _MAX_ENGINES:
                    self._synths.popitem(last=False)
                self._synths[key] = t2.wavenet.WaveNetSynthesizer(hp, B, T, cluster_size=getattr(hp, "synthesis_cluster_size", 16))
            syn = self._synths[key]
            # the live weights, not the EMA shadow: the reference's checkpoints store the live values under the shadow names
            # (wavenet_vocoder/train.py:75-83; SURVEY.md Appendix D.13), so that is what its synthesizer restores
            src = next(reversed(self._engines.values())) if self._engines else None
            if src is not None:
                syn.load_params(src.export_params())
            elif getattr(self, "_pending", None) is not None:
                syn.load_params(self._pending)
            else:
                syn.init_variables()
            initial = torch.zeros(B, dtype=torch.float32 if scalar else torch.int32, device=c.device)
            if not scalar:
                initial.fill_((hp.quantize_channels - 1) // 2)                      # mulaw_quantize(0) (wavenet.py:341-348)
            out = syn.generate(c.float().contiguous(), initial, test_inputs=test_inputs, speakers=g)
            # wavenet.py:450-456: the published y_hat is the decoded waveform in [-1, 1]
            if is_mulaw_quantize(hp.input_type):
                out = t2.audio.inv_mulaw_quantize(out.contiguous())
            elif is_mulaw(hp.input_type):
                out = t2.audio.inv_mulaw(out.contiguous())
            self.tower_y_hat = [out.reshape(B, -1)]
            self.tower_synth_upsampled_local_features = []
        return self

    def add_loss(self):
        """wavenet.py:476-519 (MaskedCrossEntropyLoss / DiscretizedMixtureLogisticLoss, tower mean)."""
        s = self._eng.loss_buf
        self.tower_loss = [s[0] / torch.clamp(s[1], min=1e-20)]
        self.loss = self.tower_loss[0]
        if self.is_evaluating:
            self.eval_loss = self.loss
        return self.loss

    def add_optimizer(self, global_step=None):
        """wavenet.py:522-613: gradients -> mean over ranks -> clip_by_norm / clip_by_value -> Adam -> EMA."""
        import torch.distributed as dist
        eng = self._eng
        if global_step is not None:
            eng.global_step = int(global_step)
        eng.backward()
        world = dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1
        if world > 1:
            dist.all_reduce(eng.grads, op=dist.ReduceOp.SUM)
        self.learning_rate = eng.optimizer_step(grad_scale=1.0 / world)
        for other in self._engines.values():                        # buffers are shared; keep counters in step
            other.global_step = eng.global_step
            other.m, other.v, other.ema, other.grads = eng.m, eng.v, eng.ema, eng.grads
            other._packed_dirty = True
        self.gradients = eng.grads
        self.optimize = None                                        # already applied (nothing left to sess.run)
        self.ema = eng.ema
        return self.learning_rate
