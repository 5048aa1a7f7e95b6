"""Host side of the H100 Tacotron-2 mel predictor (training graph). Mirrors tacotron/models/tacotron.py: the
reference's ``initialize`` + ``add_loss`` + ``add_optimizer`` become ``forward`` / ``backward`` / ``optimizer_step``."""
import ctypes
import math

import torch

from . import lib as L

N_SYMBOLS = 66


class TacoConfig(ctypes.Structure):
    _fields_ = [(n, ctypes.c_int) for n in (
        "B", "T_in", "T_out", "n_symbols", "num_mels", "embedding_dim", "enc_conv_layers", "enc_conv_kernel",
        "enc_conv_channels", "encoder_lstm_units", "attention_dim", "attention_filters", "attention_kernel", "prenet1",
        "prenet2", "decoder_lstm_units", "postnet_layers", "postnet_kernel", "postnet_channels", "clip_outputs")] + [
        (n, ctypes.c_float) for n in ("dropout_rate", "zoneout_rate", "reg_weight", "max_abs_value", "lower_bound_decay")] + [
        ("split_bf16", ctypes.c_int), ("mask_decoder", ctypes.c_int), ("cross_entropy_pos_weight", ctypes.c_float),
        ("unmasked_encoder", ctypes.c_int), ("noncumulative_weights", ctypes.c_int), ("teacher_forcing_ratio", ctypes.c_float)]


class CbhgConfig(ctypes.Structure):
    _fields_ = [(n, ctypes.c_int) for n in (
        "B", "T", "num_mels", "kernels", "conv_channels", "pool_size", "projection", "projection_kernel_size", "highwaynet_layers",
        "highway_units", "rnn_units", "num_freq", "n_priority_freq", "clip_outputs", "mask_decoder")] + [
        (n, ctypes.c_float) for n in ("max_abs_value", "lower_bound_decay", "reg_weight")] + [("split_bf16", ctypes.c_int)]


def _decay_field(hp):
    """The kernels clip outputs to [-max_abs_value - lower_bound_decay, max_abs_value]. The reference's lower bound is
    T2_output_range[0] - lower_bound_decay with T2_output_range[0] = -max_abs_value for symmetric mels and 0 otherwise
    (tacotron.py:89,176,199): the asymmetric case is expressed through the same two fields by folding max_abs_value into the decay."""
    return hp.lower_bound_decay if hp.symmetric_mels else hp.lower_bound_decay - hp.max_abs_value


def make_cbhg_config(hp, B, T, reg_weight, precision="bf16"):
    """CBHG post-processing net + linear head (tacotron.py:203-219); the shapes the CUDA path implements are checked by t2_cbhg_sizes.
    precision 'fp32-class': split bf16 hi + lo operands, forward only (include/t2b200.h, t2_cbhg_config_t.split_bf16)."""
    if precision not in ("bf16", "fp32-class"):
        raise L.T2Error("precision must be 'bf16' or 'fp32-class'")
    c = CbhgConfig()
    c.B, c.T, c.num_mels = B, T, hp.num_mels
    c.kernels, c.conv_channels, c.pool_size = hp.cbhg_kernels, hp.cbhg_conv_channels, hp.cbhg_pool_size
    c.projection, c.projection_kernel_size = hp.cbhg_projection, hp.cbhg_projection_kernel_size
    c.highwaynet_layers, c.highway_units, c.rnn_units = hp.cbhg_highwaynet_layers, hp.cbhg_highway_units, hp.cbhg_rnn_units
    c.num_freq = hp.num_freq
    c.n_priority_freq = int(2000 / (hp.sample_rate * 0.5) * hp.num_freq)
    c.clip_outputs, c.mask_decoder = int(hp.clip_outputs), int(bool(hp.mask_decoder))
    c.max_abs_value, c.lower_bound_decay, c.reg_weight = hp.max_abs_value, _decay_field(hp), reg_weight
    c.split_bf16 = int(precision == "fp32-class")
    return c


def unsupported_hparams(hp):
    """hparam-gated variants of the reference graph that change the arithmetic and that this path does NOT implement: every one
    is rejected instead of silently training a different model (SURVEY.md §8f.4). Returns a list of human-readable reasons."""
    bad = []
    def need(name, ok, why):
        if name in hp and not ok(getattr(hp, name)):
            bad.append("%s=%r (%s)" % (name, getattr(hp, name), why))
    need("outputs_per_step", lambda v: v == 1, "reduction factor r > 1: tacotron.py:141-143, helpers.py:77")
    if getattr(hp, "predict_linear", False):
        need("cbhg_pool_size", lambda v: v == 2, "CBHG max-pool width 2")
        need("cbhg_kernels", lambda v: 1 <= v <= 8, "CBHG convolution bank of at most 8 kernel sizes")
        need("cbhg_conv_channels", lambda v: v == 128, "CBHG bank of 128 channels")
        need("cbhg_highway_units", lambda v: v == 128, "128 highway units")
        need("cbhg_rnn_units", lambda v: v == 128, "128 GRU units")
    need("prenet_layers", lambda v: len(v) == 2, "2 prenet layers")
    need("decoder_layers", lambda v: v == 2, "2 decoder LSTM layers")
    need("smoothing", lambda v: not v, "smoothing normalisation instead of softmax: attention.py:72-92")
    need("batch_norm_position", lambda v: v == "after", "batch norm before the activation: modules.py:386-389")
    need("tacotron_teacher_forcing_mode", lambda v: v == "constant", "scheduled teacher forcing: helpers.py:135-169")
    need("tacotron_teacher_forcing_ratio", lambda v: 0.0 <= float(v) <= 1.0, "teacher-forcing ratio outside [0, 1]: helpers.py:121-124")
    need("synthesis_constraint", lambda v: not v, "attention window / monotonic constraint at synthesis: attention.py:201-214")
    need("tacotron_natural_eval", lambda v: not v, "evaluation that feeds the model its own predictions: helpers.py:97-100")
    if not getattr(hp, "mask_decoder", False):
        need("cross_entropy_pos_weight", lambda v: float(v) == 1.0, "the weighted stop-token loss only exists in the masked loss path")
    return bad


def make_config(hp, B, T_in, T_out, precision="bf16", teacher_forcing_ratio=None):
    """teacher_forcing_ratio: None = hparams.tacotron_teacher_forcing_ratio ('constant' mode); GTA passes 1 (helpers.py:101-102)"""
    if precision not in ("bf16", "fp32-class"):
        raise L.T2Error("precision must be 'bf16' or 'fp32-class'")
    bad = unsupported_hparams(hp)
    if bad:
        raise L.T2Error("hparams not implemented on the H100 Tacotron path (they would change the model): " + "; ".join(bad))
    c = TacoConfig()
    c.B, c.T_in, c.T_out = B, T_in, T_out
    c.n_symbols, c.num_mels, c.embedding_dim = N_SYMBOLS, hp.num_mels, hp.embedding_dim
    c.enc_conv_layers, c.enc_conv_kernel, c.enc_conv_channels = hp.enc_conv_num_layers, hp.enc_conv_kernel_size[0], hp.enc_conv_channels
    c.encoder_lstm_units = hp.encoder_lstm_units
    c.attention_dim, c.attention_filters, c.attention_kernel = hp.attention_dim, hp.attention_filters, hp.attention_kernel[0]
    c.prenet1, c.prenet2 = hp.prenet_layers
    c.decoder_lstm_units = hp.decoder_lstm_units
    c.postnet_layers, c.postnet_kernel, c.postnet_channels = hp.postnet_num_layers, hp.postnet_kernel_size[0], hp.postnet_channels
    c.clip_outputs = int(hp.clip_outputs)
    reg_weight = hp.tacotron_reg_weight
    if getattr(hp, "tacotron_scale_regularization", False):       # tacotron.py:334-338
        reg_weight *= 1.0 / (2 * hp.max_abs_value) if hp.symmetric_mels else 1.0 / hp.max_abs_value
    c.dropout_rate, c.zoneout_rate, c.reg_weight = hp.tacotron_dropout_rate, hp.tacotron_zoneout_rate, reg_weight
    c.max_abs_value, c.lower_bound_decay = hp.max_abs_value, _decay_field(hp)
    c.split_bf16 = int(precision == "fp32-class")
    c.mask_decoder = int(bool(hp.mask_decoder))
    c.cross_entropy_pos_weight = float(hp.cross_entropy_pos_weight)
    c.unmasked_encoder = int(not getattr(hp, "mask_encoder", True))               # attention.py:140-151
    c.noncumulative_weights = int(not getattr(hp, "cumulative_weights", True))    # attention.py:220-224
    ratio = float(getattr(hp, "tacotron_teacher_forcing_ratio", 1.0) if teacher_forcing_ratio is None else teacher_forcing_ratio)
    if not 0.0 <= ratio <= 1.0:
        raise L.T2Error("teacher_forcing_ratio %r outside [0, 1]" % (ratio,))
    c.teacher_forcing_ratio = ratio
    return c


class Tacotron(object):
    def __init__(self, hparams, B, T_in, T_out, device="cuda", precision="bf16", teacher_forcing_ratio=None):
        """precision 'fp32-class': every contraction of the forward and of synthesize() - convolution stacks, encoder BiLSTM, prenet,
        decoder LSTMs, attention, frame / stop projection, and with predict_linear the CBHG head and linear projection - runs on bf16
        hi + lo operand pairs with hi + lo stored activations and fp32 pre-batch-norm activations / cell states; forward / losses /
        synthesis / linear_from_mel only (include/t2b200.h, t2_taco_config_t.split_bf16 and t2_cbhg_config_t.split_bf16).
        teacher_forcing_ratio (default hparams.tacotron_teacher_forcing_ratio): below 1, every decoder step of forward() draws whether
        the next step consumes the target frame or the frame just predicted, and backward() differentiates through the fed-back frames."""
        self.hp = hparams
        self.lib = L.load()
        self.device = torch.device(device)
        self.precision = precision
        self.cfg = make_config(hparams, B, T_in, T_out, precision, teacher_forcing_ratio)
        n, pb, wb, nt = ctypes.c_longlong(), ctypes.c_longlong(), ctypes.c_longlong(), ctypes.c_int()
        L.check(self.lib.t2_taco_sizes(ctypes.byref(self.cfg), ctypes.byref(n), ctypes.byref(pb), ctypes.byref(wb), ctypes.byref(nt)))
        self.n_taco = n.value
        self.tensors = L.param_table(self.lib.t2_taco_param_info, self.cfg, nt.value)
        self.cbhg = None
        n_cb = 0
        if getattr(hparams, "predict_linear", False):       # CBHG + linear head: a second engine chained on mel_outputs (include/t2b200.h)
            self.cbhg = make_cbhg_config(hparams, B, T_out, self.cfg.reg_weight, precision)
            cn, cpb, cwb, cnt = ctypes.c_longlong(), ctypes.c_longlong(), ctypes.c_longlong(), ctypes.c_int()
            L.check(self.lib.t2_cbhg_sizes(ctypes.byref(self.cbhg), ctypes.byref(cn), ctypes.byref(cpb), ctypes.byref(cwb), ctypes.byref(cnt)))
            n_cb = cn.value
            self.cb_packed = torch.empty(cpb.value, dtype=torch.uint8, device=self.device)
            self.cb_workspace = torch.empty(cwb.value, dtype=torch.uint8, device=self.device)
            self.cb_loss = torch.zeros(2, dtype=torch.float32, device=self.device)
            self.cb_dmel = torch.zeros(B * T_out * hparams.num_mels, dtype=torch.float32, device=self.device)
            self.tensors += L.param_table(self.lib.t2_cbhg_param_info, self.cbhg, cnt.value, base=self.n_taco)
        self.n_params = n.value + n_cb
        self.params = torch.zeros(self.n_params, dtype=torch.float32, device=self.device)
        self.packed = torch.empty(pb.value, dtype=torch.uint8, device=self.device)
        self.workspace = torch.empty(wb.value, dtype=torch.uint8, device=self.device)
        self.loss_buf = torch.zeros(4, dtype=torch.float32, device=self.device)
        self.grads = self.m = self.v = None
        self.offsets = torch.tensor([t[1] for t in self.tensors] + [self.n_params], dtype=torch.int64, device=self.device)
        self.opt_scratch = torch.zeros(L.adam_scratch_floats(len(self.tensors), self.n_params), dtype=torch.float32, device=self.device)
        self.step_dev = torch.zeros(1, dtype=torch.int64, device=self.device)
        self.global_step = 0
        self.seed = int(hparams.tacotron_random_seed)
        with torch.cuda.device(self.device):
            L.check(self.lib.t2_taco_init(ctypes.byref(self.cfg), L.ptr(self.packed), L.ptr(self.workspace), L.stream_ptr()))
            if self.cbhg is not None:
                L.check(self.lib.t2_cbhg_init(ctypes.byref(self.cbhg), L.ptr(self.cb_packed), L.ptr(self.cb_workspace), L.stream_ptr()))
        self._dirty = True

    def load_params(self, params):
        flat = torch.zeros(self.n_params, dtype=torch.float32)
        for name, off, shape, _ in self.tensors:
            flat[off:off + int(math.prod(shape))] = params[name].detach().float().reshape(-1)
        self.params.copy_(flat.to(self.device))
        self._dirty = True

    def init_variables(self, seed=None):
        """fresh variables: glorot-uniform kernels / embedding, zero biases, unit batch-norm (see init.py)"""
        from . import init
        self.load_params(init.tacotron_variables(self.hp, self.tensors, seed))

    def unflatten(self, flat, trainable_only=False):
        flat = flat.detach().float().cpu()
        return {n: flat[o:o + int(math.prod(s))].reshape(s).clone() for n, o, s, tr in self.tensors if tr or not trainable_only}

    def export_params(self):
        return self.unflatten(self.params)

    def export_grads(self):
        return self.unflatten(self.grads, trainable_only=True)

    def pack(self):
        L.check(self.lib.t2_taco_pack_weights(ctypes.byref(self.cfg), L.ptr(self.params), L.ptr(self.packed), L.ptr(self.workspace), L.stream_ptr()))
        if self.cbhg is not None:
            L.check(self.lib.t2_cbhg_pack_weights(ctypes.byref(self.cbhg), L.ptr(self.params[self.n_taco:]), L.ptr(self.cb_packed),
                                                  L.ptr(self.cb_workspace), L.stream_ptr()))
        self._dirty = False

    def forward(self, inputs, input_lengths, mel_targets, stop_targets, training=True, seed=None, targets_lengths=None, linear_targets=None):
        """targets_lengths: int32 [B] device tensor, required when hparams.mask_decoder (masked losses, modules.py:412-455);
        linear_targets: fp32 [B, T_out, num_freq], required in training when hparams.predict_linear (tacotron.py:45-46)"""
        if self._dirty:
            self.pack()
        if self.cfg.mask_decoder:
            if targets_lengths is None:
                raise L.T2Error("Model set to mask paddings but no targets lengths provided for the mask!")
            L.check(self.lib.t2_taco_set_target_lengths(ctypes.byref(self.cfg), L.ptr(self.workspace), L.ptr(targets_lengths), L.stream_ptr()))
        self._last = (inputs, input_lengths, mel_targets, stop_targets)
        self._last_seed = self.seed if seed is None else seed
        L.check(self.lib.t2_taco_forward(ctypes.byref(self.cfg), L.ptr(self.params), L.ptr(self.packed), L.ptr(self.workspace),
                                         L.ptr(inputs), L.ptr(input_lengths), L.ptr(mel_targets), L.ptr(stop_targets),
                                         L.ptr(self.loss_buf), int(training), ctypes.c_ulonglong(self._last_seed),
                                         L.ptr(self.step_dev), L.stream_ptr()))
        if self.cbhg is not None:
            if training and linear_targets is None:
                raise L.T2Error("Model is set to use post processing to predict linear spectrograms in training but no linear targets given!")
            if self.cfg.mask_decoder:
                L.check(self.lib.t2_cbhg_set_target_lengths(ctypes.byref(self.cbhg), L.ptr(self.cb_workspace), L.ptr(targets_lengths), L.stream_ptr()))
            self._last_linear = linear_targets
            mel = self.workspace_tensor("mel_outputs")
            L.check(self.lib.t2_cbhg_forward(ctypes.byref(self.cbhg), L.ptr(self.params[self.n_taco:]), L.ptr(self.cb_packed), L.ptr(self.cb_workspace),
                                             L.ptr(mel), L.ptr(linear_targets), L.ptr(self.cb_loss), int(training), L.stream_ptr()))
        return self.loss_buf

    def backward(self):
        if self.grads is None:
            self.grads = torch.zeros_like(self.params)
        inputs, input_lengths, mel_targets, stop_targets = self._last
        extra = None
        if self.cbhg is not None:      # the post-processing net first: it yields the extra gradient on mel_outputs
            L.check(self.lib.t2_cbhg_backward(ctypes.byref(self.cbhg), L.ptr(self.params[self.n_taco:]), L.ptr(self.cb_packed), L.ptr(self.cb_workspace),
                                              L.ptr(self.workspace_tensor("mel_outputs")), L.ptr(self.grads[self.n_taco:]), L.ptr(self.cb_dmel),
                                              L.stream_ptr()))
            extra = self.cb_dmel
        L.check(self.lib.t2_taco_backward_ex(ctypes.byref(self.cfg), L.ptr(self.params), L.ptr(self.packed), L.ptr(self.workspace),
                                             L.ptr(inputs), L.ptr(input_lengths), L.ptr(mel_targets), L.ptr(stop_targets),
                                             L.ptr(self.grads), L.ptr(extra), ctypes.c_ulonglong(self._last_seed), L.ptr(self.step_dev),
                                             L.stream_ptr()))
        return self.grads

    def linear_outputs(self):
        """[B, T_out, num_freq] fp32 (clipped) of the last forward (predict_linear)"""
        p, cnt = ctypes.c_void_p(), ctypes.c_longlong()
        L.check(self.lib.t2_cbhg_workspace_tensor(ctypes.byref(self.cbhg), L.ptr(self.cb_workspace), b"linear_outputs", ctypes.byref(p), ctypes.byref(cnt)))
        off = p.value - self.cb_workspace.data_ptr()
        nfp = (self.hp.num_freq + 7) // 8 * 8
        return self.cb_workspace[off:off + cnt.value * 4].view(torch.float32).reshape(self.cfg.B, self.cfg.T_out, nfp)[:, :, :self.hp.num_freq]

    def linear_from_mel(self, mel):
        """Inference-mode post-processing net on finished mel_outputs [B, T, num_mels] (synthesis: tacotron.py:203-219 with
        is_training = False) -> linear spectrogram [B, T, num_freq]. Runs a CBHG engine sized for this (B, T)."""
        if self._dirty:
            self.pack()
        B0, T = int(mel.shape[0]), int(mel.shape[1])
        B = (B0 + 3) // 4 * 4                                   # the recurrent kernel takes items in fours; rows are independent here
        x = torch.zeros(B, max(T, 2), self.hp.num_mels, dtype=torch.float32, device=self.device)
        x[:B0, :T] = mel.float()
        cfg = make_cbhg_config(self.hp, B, max(T, 2), 0.0, self.precision)
        cfg.mask_decoder = 0
        pb, wb = ctypes.c_longlong(), ctypes.c_longlong()
        L.check(self.lib.t2_cbhg_sizes(ctypes.byref(cfg), None, ctypes.byref(pb), ctypes.byref(wb), None))
        packed = torch.empty(pb.value, dtype=torch.uint8, device=self.device)
        ws = torch.empty(wb.value, dtype=torch.uint8, device=self.device)
        prm = self.params[self.n_taco:]
        L.check(self.lib.t2_cbhg_init(ctypes.byref(cfg), L.ptr(packed), L.ptr(ws), L.stream_ptr()))
        L.check(self.lib.t2_cbhg_pack_weights(ctypes.byref(cfg), L.ptr(prm), L.ptr(packed), L.ptr(ws), L.stream_ptr()))
        L.check(self.lib.t2_cbhg_forward(ctypes.byref(cfg), L.ptr(prm), L.ptr(packed), L.ptr(ws), L.ptr(x), L.ptr(None), L.ptr(None), 0, L.stream_ptr()))
        p, cnt = ctypes.c_void_p(), ctypes.c_longlong()
        L.check(self.lib.t2_cbhg_workspace_tensor(ctypes.byref(cfg), L.ptr(ws), b"linear_outputs", ctypes.byref(p), ctypes.byref(cnt)))
        off = p.value - ws.data_ptr()
        nfp = (self.hp.num_freq + 7) // 8 * 8
        return ws[off:off + cnt.value * 4].view(torch.float32).reshape(B, max(T, 2), nfp)[:B0, :T, :self.hp.num_freq].clone()

    def synthesize(self, inputs, input_lengths, max_iters=None, chunk=64, seed=None):
        """Free-running synthesis (TacoTestHelper, helpers.py:6-59): feed back the predicted frame, stop after the first
        step at which EVERY batch row has round(sigmoid(stop)) == 1 (r = 1) or at max_iters (<= T_out of this instance).
        The stop rule is evaluated on the host between chunks of `chunk` steps; frames decoded past the stop step are
        discarded, which is what the reference's dynamic_decode returns. Returns dict(mel_outputs [B, T, M],
        decoder_output [B, T, M], alignments [B, T, T_in], stop_token_prediction [B, T] (sigmoid), T)."""
        if self._dirty:
            self.pack()
        To = self.cfg.T_out if max_iters is None else min(max_iters, self.cfg.T_out)
        seed = self.seed if seed is None else seed
        cfg, B, M = ctypes.byref(self.cfg), self.cfg.B, self.cfg.num_mels
        L.check(self.lib.t2_taco_infer_begin(cfg, L.ptr(self.params), L.ptr(self.packed), L.ptr(self.workspace), L.ptr(inputs),
                                             L.ptr(input_lengths), L.stream_ptr()))
        rows = self.workspace_tensor("projection_rows", (self.cfg.T_out, B, 128))
        t, T_used = 0, To
        while t < To:
            t_end = min(t + chunk, To)
            L.check(self.lib.t2_taco_infer_steps(cfg, L.ptr(self.params), L.ptr(self.packed), L.ptr(self.workspace),
                                                 L.ptr(input_lengths), t, t_end, ctypes.c_ulonglong(seed), L.stream_ptr()))
            done = (rows[t:t_end, :, M] > 0).all(dim=1)      # round(sigmoid(z)) == 1  <=>  z > 0 (half rounds to even: 0)
            hit = torch.nonzero(done)
            if hit.numel():
                T_used = t + int(hit[0, 0]) + 1
                break
            t = t_end
        L.check(self.lib.t2_taco_infer_finish(cfg, L.ptr(self.params), L.ptr(self.packed), L.ptr(self.workspace), T_used, L.stream_ptr()))
        Ti = self.cfg.T_in
        return {"T": T_used,
                "mel_outputs": self.workspace_tensor("mel_outputs", (B, T_used, M)).clone(),
                "decoder_output": self.workspace_tensor("decoder_output", (B, T_used, M)).clone(),
                "stop_token_prediction": torch.sigmoid(self.workspace_tensor("stop_logits", (B, T_used))),
                "alignments": self.workspace_tensor("alignments", (self.cfg.T_out, B, Ti))[:T_used].transpose(0, 1).clone()}

    def capture(self, inputs, input_lengths, mel_targets, stop_targets, linear_targets=None, targets_lengths=None):
        """Capture pack + forward + backward (~7.5k kernel nodes at B=32, T_out=800) into one CUDA graph over static inputs."""
        self._static = (inputs, input_lengths, mel_targets, stop_targets)
        self._static_kw = dict(linear_targets=linear_targets, targets_lengths=targets_lengths)
        if self.grads is None:
            self.grads = torch.zeros_like(self.params)
        side = torch.cuda.Stream(device=self.device)
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            self.pack()
            self.forward(*self._static, **self._static_kw)
            self.backward()
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        self._graph = torch.cuda.CUDAGraph()
        n0 = self.lib.t2_launch_count()
        with torch.cuda.graph(self._graph):
            self.step_dev.add_(1)
            self.pack()
            self.forward(*self._static, **self._static_kw)
            self.backward()
        self._fwd_bwd_launches = self.lib.t2_launch_count() - n0
        return self._graph

    def train_step(self, inputs=None, input_lengths=None, mel_targets=None, stop_targets=None, world_size=1, linear_targets=None,
                   targets_lengths=None):
        """forward + losses + backward (+ NCCL all-reduce) + clip_by_global_norm + Adam (tacotron.py:406-437 order)."""
        if getattr(self, "_graph", None) is not None:
            for dst, src in zip(self._static + (self._static_kw["linear_targets"], self._static_kw["targets_lengths"]),
                                (inputs, input_lengths, mel_targets, stop_targets, linear_targets, targets_lengths)):
                if src is not None and dst is not None and src is not dst:
                    dst.copy_(src, non_blocking=True)
            self._graph.replay()
        else:
            n0 = self.lib.t2_launch_count()
            self.step_dev.add_(1)
            self.forward(inputs, input_lengths, mel_targets, stop_targets, linear_targets=linear_targets, targets_lengths=targets_lengths)
            self.backward()
            self._fwd_bwd_launches = self.lib.t2_launch_count() - n0
        if world_size > 1:
            import torch.distributed as dist
            dist.all_reduce(self.grads, op=dist.ReduceOp.SUM)
        n0 = self.lib.t2_launch_count()
        self.optimizer_step(grad_scale=1.0 / world_size)
        self._opt_launches = self.lib.t2_launch_count() - n0
        return self.loss_buf

    @property
    def launches_per_step(self):
        """kernels of libt2b200 per optimisation step (graph replays re-launch the captured ones)"""
        return getattr(self, "_fwd_bwd_launches", 0) + getattr(self, "_opt_launches", 0)

    def learning_rate(self):
        hp = self.hp
        if not hp.tacotron_decay_learning_rate:
            return hp.tacotron_initial_learning_rate
        lr = hp.tacotron_initial_learning_rate * hp.tacotron_decay_rate ** (
            (self.global_step - hp.tacotron_start_decay) / hp.tacotron_decay_steps)
        return min(max(lr, hp.tacotron_final_learning_rate), hp.tacotron_initial_learning_rate)

    def optimizer_step(self, grad_scale=1.0):
        """clip_by_global_norm(1.0) + Adam (tacotron.py:393,429-437) on the flat buffers."""
        hp = self.hp
        if self.m is None:
            self.m = torch.zeros_like(self.params)
            self.v = torch.zeros_like(self.params)
        lr = self.learning_rate()
        if getattr(hp, "tacotron_fine_tuning", False):
            # tacotron.py:401: gradients are only computed for variables without 'inputs_embedding' / 'encoder_' in their names; the
            # frozen tensors lead the flat buffer, so zero their gradient (they drop out of the global norm) and first moment (no update)
            end = next(t[1] for t in self.tensors if not (t[0].startswith("inputs_embedding") or t[0].startswith("encoder_")))
            self.grads[:end].zero_()
            self.m[:end].zero_()
        L.check(self.lib.t2_adam_step(
            L.ptr(self.params), L.ptr(self.grads), L.ptr(self.m), L.ptr(self.v), L.ptr(None), L.ptr(self.offsets),
            len(self.tensors), ctypes.c_longlong(self.n_params), ctypes.c_float(lr), ctypes.c_float(hp.tacotron_adam_beta1),
            ctypes.c_float(hp.tacotron_adam_beta2), ctypes.c_float(hp.tacotron_adam_epsilon), self.global_step + 1,
            ctypes.c_float(grad_scale), ctypes.c_float(0.0), ctypes.c_float(0.0),
            ctypes.c_float(1.0 if hp.tacotron_clip_gradients else 0.0), ctypes.c_float(0.0), L.ptr(self.opt_scratch), L.stream_ptr()))
        self.global_step += 1
        self._dirty = True
        return lr

    def workspace_tensor(self, name, shape=None):
        p, cnt, eb = ctypes.c_void_p(), ctypes.c_longlong(), ctypes.c_int()
        L.check(self.lib.t2_taco_workspace_tensor(ctypes.byref(self.cfg), L.ptr(self.workspace), name.encode(), ctypes.byref(p),
                                                  ctypes.byref(cnt), ctypes.byref(eb)))
        off = p.value - self.workspace.data_ptr()
        t = self.workspace[off:off + cnt.value * eb.value].view(torch.bfloat16 if eb.value == 2 else torch.float32)
        if shape is None:
            return t
        n = 1
        for d in shape:
            n *= d
        return t[:n].reshape(shape)        # compact results (synthesis) use a prefix of the buffer

    def rng_uniform(self, stream_id, n, seed=None, first_index=0):
        """The U[0,1) draws behind the in-kernel dropout / zoneout masks of hash stream `stream_id` (include/t2b200.h,
        t2_rng_uniform_f32) for the step that ran with `seed` (default: this model's seed + the device step counter)."""
        if seed is None:
            seed = getattr(self, "_last_seed", self.seed) + int(self.step_dev.item())
        out = torch.empty(n, dtype=torch.float32, device=self.device)
        L.check(self.lib.t2_rng_uniform_f32(ctypes.c_ulonglong(seed), ctypes.c_uint(stream_id), ctypes.c_longlong(first_index),
                                            ctypes.c_longlong(n), L.ptr(out), L.stream_ptr()))
        return out

    def teacher_forcing_choices(self):
        """bool [T_out] of the last forward at a teacher-forcing ratio < 1: element t is True when step t + 1 consumed the target
        frame t, False when it consumed the frame step t predicted (the draw of element t, hash stream 40, is below the ratio)"""
        return self.workspace_tensor("teacher_forced").view(torch.int32) != 0

    def losses(self):
        b, a, s, r = self.loss_buf.tolist()
        out = {"before": b, "after": a, "stop": s, "reg": r, "linear": 0.0}
        if self.cbhg is not None:
            lin, rc = self.cb_loss.tolist()
            out["linear"], out["reg"] = lin, r + rc       # one regulariser over all variables (tacotron.py:343-345)
        out["total"] = out["before"] + out["after"] + out["stop"] + out["reg"] + out["linear"]
        return out
