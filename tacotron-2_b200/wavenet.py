"""Host side of the H100 WaveNet vocoder: owns device buffers (torch tensors) and drives libt2b200.so.

Mirrors the reference's model object (wavenet_vocoder/models/wavenet.py): ``WaveNet(hparams)`` then
``initialize`` / ``step`` (forward), ``add_loss`` (loss) and ``add_optimizer`` (Adam + clipping + EMA) collapse into
``forward`` / ``backward`` / ``optimizer_step`` / ``train_step`` here, because there is no graph to build.
All arithmetic runs in the CUDA library; torch is used for allocation, streams, CUDA graphs and NCCL.
"""
import ctypes
import math

import torch

from . import lib as L


class WnConfig(ctypes.Structure):
    _fields_ = [
        ("layers", ctypes.c_int), ("stacks", ctypes.c_int), ("residual_channels", ctypes.c_int),
        ("gate_channels", ctypes.c_int), ("skip_out_channels", ctypes.c_int), ("kernel_size", ctypes.c_int),
        ("cin_channels", ctypes.c_int), ("out_channels", ctypes.c_int), ("quantize_channels", ctypes.c_int),
        ("input_type", ctypes.c_int), ("legacy", ctypes.c_int), ("residual_legacy", ctypes.c_int),
        ("upsample_type", ctypes.c_int), ("n_upsample", ctypes.c_int), ("upsample_scales", ctypes.c_int * 4),
        ("freq_axis_kernel_size", ctypes.c_int), ("dropout", ctypes.c_float), ("log_scale_min", ctypes.c_float),
        ("B", ctypes.c_int), ("T", ctypes.c_int), ("Tc", ctypes.c_int), ("c_pre_upsampled", ctypes.c_int),
        ("log_scale_min_gauss", ctypes.c_float), ("cdf_loss", ctypes.c_int), ("split_bf16", ctypes.c_int),
        ("gin_channels", ctypes.c_int), ("n_speakers", ctypes.c_int),
        ("upsample_activation", ctypes.c_int), ("leaky_alpha", ctypes.c_float),
    ]


class WnSizes(ctypes.Structure):
    _fields_ = [("n_params", ctypes.c_longlong), ("packed_bytes", ctypes.c_longlong),
                ("workspace_bytes", ctypes.c_longlong), ("n_tensors", ctypes.c_int)]


_INPUT_TYPES = {"raw": 0, "mulaw": 1, "mulaw-quantize": 2}
_UPSAMPLE_TYPES = {"SubPixel": 0, "2D": 1, "1D": 2}
# activation after each learnable upsampling layer (wavenet.py:197-203); None = linear
_UPSAMPLE_ACTIVATIONS = {"Relu": 0, "relu": 0, "RELU": 0, "LeakyRelu": 1, None: 2}


def _leaky_alpha_ok(v):
    try:
        a = float(v)
    except (TypeError, ValueError):
        return False
    return 0.0 <= a <= 1.0          # NaN fails both comparisons


def unsupported_hparams(hp):
    """hparam-gated variants of the reference WaveNet that change the arithmetic and are NOT implemented here (SURVEY.md §8f.4)"""
    bad = []
    def need(name, ok, why):
        if name in hp and not ok(getattr(hp, name)):
            bad.append("%s=%r (%s)" % (name, getattr(hp, name), why))
    need("wavenet_weight_normalization", lambda v: not v, "weight normalisation with data-dependent init: modules.py:44-177")
    need("use_bias", lambda v: bool(v), "bias-free convolutions")
    if (getattr(hp, "gin_channels", None) or 0) > 0:        # global (speaker) conditioning through gc_embedding
        need("use_speaker_embedding", lambda v: bool(v),
             "speaker ids fed straight into the gin convolution without an embedding: wavenet.py:151-158")
        need("n_speakers", lambda v: v is not None and v >= 1, "gin_channels > 0 needs n_speakers >= 1")
    need("kernel_size", lambda v: v in (2, 3, 4), "kernel_size 2, 3 or 4")
    need("upsample_type", lambda v: v in _UPSAMPLE_TYPES or v == "NearestNeighbor", "Resize upsampler: modules.py:657-693")
    need("upsample_activation", lambda v: v in _UPSAMPLE_ACTIVATIONS, "Relu | LeakyRelu | None: wavenet.py:197-203")
    if getattr(hp, "upsample_activation", None) == "LeakyRelu":
        need("leaky_alpha", _leaky_alpha_ok, "LeakyRelu slope in [0, 1] (max(alpha * x, x) is leaky_relu only there)")
    if getattr(hp, "upsample_type", None) != "1D":             # ConvTranspose1D has no frequency axis (modules.py:697-733)
        need("freq_axis_kernel_size", lambda v: v == 3, "freq_axis_kernel_size 3")
    need("input_type", lambda v: v in _INPUT_TYPES, "raw | mulaw | mulaw-quantize")
    need("wavenet_synth_debug", lambda v: not v, "teacher-forced synthesis debugging from wavenet_debug_wavs: synthesizer.py:54-57,85-97")
    need("wavenet_natural_eval", lambda v: not v, "free-running evaluation: wavenet.py:386 (evaluation here is teacher forced)")
    return bad


def make_config(hp, B, T, c_pre_upsampled=False, dropout=None, precision="bf16"):
    bad = unsupported_hparams(hp)
    if bad:
        raise L.T2Error("hparams not implemented on the H100 WaveNet path (they would change the model): " + "; ".join(bad))
    cfg = WnConfig()
    cfg.layers, cfg.stacks = hp.layers, hp.stacks
    cfg.residual_channels, cfg.gate_channels, cfg.skip_out_channels = (
        hp.residual_channels, hp.gate_channels, hp.skip_out_channels)
    cfg.kernel_size = hp.kernel_size
    cfg.cin_channels = max(hp.cin_channels, 0)
    cfg.out_channels, cfg.quantize_channels = hp.out_channels, hp.quantize_channels
    cfg.input_type = _INPUT_TYPES[hp.input_type]
    cfg.legacy, cfg.residual_legacy = int(hp.legacy), int(hp.residual_legacy)
    if hp.upsample_type == "NearestNeighbor":     # non-learnable repeat (modules.py:524-536, wavenet.py:165-167): done by nn_upsample() below
        c_pre_upsampled = True
    elif hp.upsample_type not in _UPSAMPLE_TYPES:
        raise L.T2Error("upsample_type %r is not implemented on the H100 path" % hp.upsample_type)
    cfg.upsample_type = _UPSAMPLE_TYPES.get(hp.upsample_type, 0)
    act = getattr(hp, "upsample_activation", "Relu")
    cfg.upsample_activation = _UPSAMPLE_ACTIVATIONS[act]
    cfg.leaky_alpha = float(hp.leaky_alpha) if act == "LeakyRelu" else 0.0
    scales = list(hp.upsample_scales)
    cfg.n_upsample = len(scales)
    for i, s in enumerate(scales):
        cfg.upsample_scales[i] = s
    cfg.freq_axis_kernel_size = hp.freq_axis_kernel_size
    cfg.dropout = hp.wavenet_dropout if dropout is None else dropout
    cfg.log_scale_min = hp.log_scale_min
    cfg.log_scale_min_gauss = getattr(hp, "log_scale_min_gauss", -7.0)
    cfg.cdf_loss = int(getattr(hp, "cdf_loss", False))
    if precision not in ("bf16", "fp32-class"):
        raise L.T2Error("precision must be 'bf16' or 'fp32-class'")
    cfg.split_bf16 = int(precision == "fp32-class")
    if (getattr(hp, "gin_channels", None) or 0) > 0:
        cfg.gin_channels, cfg.n_speakers = hp.gin_channels, hp.n_speakers
    cfg.B, cfg.T = B, T
    hop = 1
    for s in scales:
        hop *= s
    cfg.c_pre_upsampled = int(c_pre_upsampled)
    if cfg.cin_channels > 0 and not c_pre_upsampled:
        if T % hop:
            raise L.T2Error("T=%d is not a multiple of prod(upsample_scales)=%d" % (T, hop))
        cfg.Tc = T // hop
    else:
        cfg.Tc = T
    return cfg


def param_table(cfg):
    """[(name, offset, shape)] + n_params of the flat parameter buffer for a config: host-only library calls (no CUDA device needed)"""
    lib = L.load()
    sz = WnSizes()
    L.check(lib.t2_wn_sizes(ctypes.byref(cfg), ctypes.byref(sz)))
    return L.param_table(lib.t2_wn_param_info, cfg, sz.n_tensors, trainable=False), sz.n_params


def grad_buckets(tensors, n_layers, n_params, n_groups):
    """[(start, end)] element ranges of the flat gradient buffer for the overlapped data-parallel all-reduce: one per layer group (final
    after that group's weight-gradient launch) followed by the ranges outside the residual stack (input conv; head + upsampling net:
    final after the join). Together they cover [0, n_params) exactly once."""
    off = {t[0]: t[1] for t in tensors}
    first = lambda l: off["ResidualConv1DGLU_%d/residual_block_causal_conv/kernel" % l]
    stack_end = off["final_convolution_1/kernel"]
    bounds = [first(n_layers * g // n_groups) for g in range(n_groups)] + [stack_end]
    groups = [(bounds[g], bounds[g + 1]) for g in range(n_groups)]
    rest = [(0, first(0)), (stack_end, n_params)]
    return groups, [r for r in rest if r[1] > r[0]]


def speaker_ids(speakers, B, n_speakers):
    """speaker ids ([B, 1] or [B] ints, tensor or sequence) -> int32 [B] on the host; raises ValueError on a bad shape or an id outside
    [0, n_speakers), before anything reaches the device"""
    ids = torch.as_tensor(speakers).detach().cpu().reshape(-1)
    if ids.numel() != B or ids.is_floating_point() or ids.is_complex():
        raise ValueError("speaker ids must be %d integers ([B] or [B, 1]), got %s %s" % (B, tuple(torch.as_tensor(speakers).shape), ids.dtype))
    bad = [int(v) for v in ids.tolist() if not 0 <= int(v) < n_speakers]
    if bad:
        raise ValueError("speaker id(s) %s outside [0, n_speakers=%d)" % (bad, n_speakers))
    return ids.to(torch.int32)


def nn_upsample(hp, c, T):
    """NearestNeighborUpsample (modules.py:524-536: tf.image.resize_images(method=NEAREST) by the hop size along time):
    c fp32 [B, cin, Tc] -> the channels-last pre-upsampled layout [B, T, cin] the engine takes with c_pre_upsampled = 1"""
    hop = hp.hop_size
    up = c.transpose(1, 2).repeat_interleave(hop, dim=1)
    if up.shape[1] < T:
        raise L.T2Error("conditioning of %d frames x hop %d is shorter than T=%d" % (c.shape[2], hop, T))
    return up[:, :T].contiguous()


class WaveNet(object):
    """H100 WaveNet (train path). Parameters live in ONE flat fp32 buffer in TensorFlow variable layouts."""

    def __init__(self, hparams, B, T, device="cuda", c_pre_upsampled=False, dropout=None, training=True, precision="bf16"):
        """precision: 'bf16' (training / benchmark path: bf16 operands and stored activations, fp32 accumulate) or 'fp32-class'
        (forward + loss only: every activation and weight travels as a bf16 hi + lo pair, dropout forced off)."""
        self.hp = hparams
        self.lib = L.load()
        self.device = torch.device(device)
        self.precision = precision
        if precision == "fp32-class":
            dropout = 0.0
        self.cfg = make_config(hparams, B, T, c_pre_upsampled, dropout, precision)
        self.training = training
        sz = WnSizes()
        L.check(self.lib.t2_wn_sizes(ctypes.byref(self.cfg), ctypes.byref(sz)))
        self.sizes = sz
        self.n_params = sz.n_params
        self.params = torch.zeros(sz.n_params, dtype=torch.float32, device=self.device)
        self.packed = torch.empty(sz.packed_bytes, dtype=torch.uint8, device=self.device)
        self.workspace = torch.empty(sz.workspace_bytes, dtype=torch.uint8, device=self.device)
        self.loss_buf = torch.zeros(2, dtype=torch.float32, device=self.device)
        self.grads = self.m = self.v = self.ema = None
        self.tensors = L.param_table(self.lib.t2_wn_param_info, self.cfg, sz.n_tensors, trainable=False)  # (name, offset, shape)
        offs = [t[1] for t in self.tensors] + [sz.n_params]
        self.offsets = torch.tensor(offs, dtype=torch.int64, device=self.device)
        self.opt_scratch = torch.zeros(L.adam_scratch_floats(sz.n_tensors, sz.n_params), dtype=torch.float32, device=self.device)
        self.global_step = 0
        self.seed = int(hparams.wavenet_random_seed)
        self.step_dev = torch.zeros(1, dtype=torch.int64, device=self.device)  # added to the dropout seed on device
        self._spk = torch.zeros(B, dtype=torch.int32, device=self.device) if self.cfg.gin_channels > 0 else None
        self._graph = None
        with torch.cuda.device(self.device):
            L.check(self.lib.t2_wn_init(ctypes.byref(self.cfg), L.ptr(self.packed), L.ptr(self.workspace),
                                        L.stream_ptr()))
        self._packed_dirty = True

    # ---- parameters --------------------------------------------------------------------------------------
    def load_params(self, params):
        """params: {TF-style name: tensor in TF layout}."""
        flat = torch.zeros(self.n_params, dtype=torch.float32)
        for name, off, shape in self.tensors:
            t = params[name].detach().to(torch.float32).reshape(-1)
            n = int(math.prod(shape))
            assert t.numel() == n, "%s: expected %s got %s" % (name, shape, tuple(params[name].shape))
            flat[off:off + n] = t
        self.params.copy_(flat.to(self.device))
        self._packed_dirty = True

    def init_variables(self, seed=None):
        """fresh variables: glorot-uniform kernels, zero biases, NN_init upsampling kernels (see init.py)"""
        from . import init
        self.load_params(init.wavenet_variables(self.hp, self.tensors, seed))

    def unflatten(self, flat):
        flat = flat.detach().float().cpu()
        return {name: flat[off:off + int(math.prod(shape))].reshape(shape).clone() for name, off, shape in self.tensors}

    def export_params(self):
        return self.unflatten(self.params)

    def export_grads(self):
        return self.unflatten(self.grads)

    def pack(self):
        L.check(self.lib.t2_wn_pack_weights(ctypes.byref(self.cfg), L.ptr(self.params), L.ptr(self.packed),
                                            L.ptr(self.workspace), L.stream_ptr()))
        self._packed_dirty = False

    def set_speakers(self, speakers):
        """gin_channels > 0: speaker ids ([B] or [B, 1] ints) of the following forwards, or None for no speaker term (the reference
        skips it when g is None). The ids are validated here and copied into the workspace, so a captured step uses the ids set last."""
        if self._spk is None:
            raise L.T2Error("speaker ids need gin_channels > 0")
        if speakers is None:
            L.check(self.lib.t2_wn_set_speakers(ctypes.byref(self.cfg), L.ptr(self.workspace), None, L.stream_ptr()))
            return
        self._spk.copy_(speaker_ids(speakers, self.cfg.B, self.cfg.n_speakers))
        L.check(self.lib.t2_wn_set_speakers(ctypes.byref(self.cfg), L.ptr(self.workspace), L.ptr(self._spk), L.stream_ptr()))

    # ---- compute -----------------------------------------------------------------------------------------
    def forward(self, x, c, targets, lengths, logits=None, save_for_backward=True, seed=None, speakers=None):
        """x: int32 [B,T] (mulaw-quantize) or fp32 [B,T]; c: fp32 [B,cin,Tc]; speakers: ids [B] / [B, 1] (gin_channels > 0; None keeps
        the ids of the last set_speakers, initially none); returns loss_buf (sum, normaliser)."""
        if speakers is not None:
            self.set_speakers(speakers)
        if self._packed_dirty:
            self.pack()
        if self.hp.upsample_type == "NearestNeighbor" and c is not None and c.dim() == 3 and c.shape[1] == self.cfg.cin_channels and c.shape[2] != self.cfg.T:
            c = nn_upsample(self.hp, c, self.cfg.T)
        self._last_x, self._last_c = x, c
        self._last_seed = self.seed if seed is None else seed
        L.check(self.lib.t2_wn_forward(ctypes.byref(self.cfg), L.ptr(self.params), L.ptr(self.packed),
                                       L.ptr(self.workspace), L.ptr(x), L.ptr(c), L.ptr(targets), L.ptr(lengths),
                                       L.ptr(self.loss_buf), L.ptr(logits), int(save_for_backward),
                                       ctypes.c_ulonglong(self._last_seed), L.ptr(self.step_dev), L.stream_ptr()))
        return self.loss_buf

    def backward(self, phase=-1, n_groups=1):
        """phase -1: the whole backward. Phased form (data-parallel overlap, include/t2b200.h t2_wn_backward_phased): 0 = data-gradient
        chain + head + conditioning tails, 1 + g = weight gradients of layer group g, 100 = join of the library's side stream."""
        if self.grads is None:
            self.grads = torch.zeros_like(self.params)
        L.check(self.lib.t2_wn_backward_phased(ctypes.byref(self.cfg), L.ptr(self.params), L.ptr(self.packed),
                                               L.ptr(self.workspace), L.ptr(self._last_x), L.ptr(self._last_c),
                                               L.ptr(self.grads), ctypes.c_ulonglong(self._last_seed),
                                               L.ptr(self.step_dev), int(phase), int(n_groups), L.stream_ptr()))
        return self.grads

    def grad_buckets(self, n_groups):
        return grad_buckets(self.tensors, self.cfg.layers, self.n_params, n_groups)

    # ---- training step (the call a user makes) -----------------------------------------------------------
    def capture(self, x, c, targets, lengths, overlap_groups=1):
        """Capture pack + forward + backward into CUDA graph(s) over STATIC input tensors (x, c, targets, lengths are
        the buffers later steps must copy into). Adam runs outside the graph (its bias correction changes per step).
        overlap_groups > 1 (data parallel): the step is captured as `overlap_groups` graphs cut after each layer group's
        weight-gradient GEMM, so that train_step can start that group's NCCL all-reduce (eagerly, on the process group's stream)
        while the next graph computes the next group (VERDICT r1: the monolithic all-reduce after the graph was fully exposed)."""
        self._static = (x, c, targets, lengths)
        if self.grads is None:
            self.grads = torch.zeros_like(self.params)
        G = max(1, int(overlap_groups))
        side = torch.cuda.Stream(device=self.device)
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):  # warm-up outside capture (sets kernel attributes, loads modules)
            self.pack()
            self.forward(x, c, targets, lengths)
            self.backward()
            if G > 1:
                self.backward(0, G)
                self.backward(100, G)
                for g in range(G):
                    self.backward(1 + g, G)
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        n0 = self.lib.t2_launch_count()
        self._graphs = []
        if G == 1:
            self._graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(self._graph):
                self.step_dev.add_(1)
                self.pack()
                self.forward(x, c, targets, lengths)
                self.backward()
        else:
            pool = None
            for g in range(G):
                gr = torch.cuda.CUDAGraph()
                with torch.cuda.graph(gr, pool=pool):
                    if g == 0:
                        self.step_dev.add_(1)
                        self.pack()
                        self.forward(x, c, targets, lengths)
                        self.backward(0, G)
                        # every captured graph must end with all forked streams joined: the library's side stream (conditioning
                        # tails forked in phase 0) is joined HERE, inside graph 0, not after the last group
                        self.backward(100, G)
                    self.backward(1 + g, G)
                pool = gr.pool()
                self._graphs.append(gr)
            self._graph = self._graphs[0]
            self._buckets = self.grad_buckets(G)
        self._fwd_bwd_launches = self.lib.t2_launch_count() - n0
        return self._graph

    def train_step(self, x=None, c=None, targets=None, lengths=None, world_size=1, process_group=None, speakers=None):
        """One optimisation step: forward + loss + backward (+ gradient all-reduce) + clip + Adam + EMA.
        With a captured graph, non-None arguments are copied into the static buffers first. speakers: as in forward."""
        if speakers is not None:
            self.set_speakers(speakers)
        if self._graph is not None and getattr(self, "_graphs", None):
            import torch.distributed as dist
            for dst, src in zip(self._static, (x, c, targets, lengths)):
                if src is not None and src is not dst:
                    dst.copy_(src, non_blocking=True)
            groups, rest = self._buckets
            works = []
            for gr, (a, b) in zip(self._graphs, groups):
                gr.replay()
                if world_size > 1:   # starts when this graph has finished, overlaps the next graph (the PG's own stream)
                    works.append(dist.all_reduce(self.grads[a:b], op=dist.ReduceOp.SUM, group=process_group, async_op=True))
            if world_size > 1:
                for a, b in rest:
                    works.append(dist.all_reduce(self.grads[a:b], op=dist.ReduceOp.SUM, group=process_group, async_op=True))
                for w in works:
                    w.wait()
            n0 = self.lib.t2_launch_count()
            self.optimizer_step(grad_scale=1.0 / world_size)
            self._opt_launches = self.lib.t2_launch_count() - n0
            return self.loss_buf
        if self._graph is not None:
            for dst, src in zip(self._static, (x, c, targets, lengths)):
                if src is not None and src is not dst:
                    dst.copy_(src, non_blocking=True)
            self._graph.replay()
        else:
            n0 = self.lib.t2_launch_count()
            self.step_dev.add_(1)
            self.forward(x, c, targets, lengths)
            self.backward()
            self._fwd_bwd_launches = self.lib.t2_launch_count() - n0
        if world_size > 1:
            import torch.distributed as dist
            # the reference averages tower gradients, THEN clips, THEN applies Adam (wavenet.py:561-593)
            dist.all_reduce(self.grads, op=dist.ReduceOp.SUM, group=process_group)
        n0 = self.lib.t2_launch_count()
        self.optimizer_step(grad_scale=1.0 / world_size)
        self._opt_launches = self.lib.t2_launch_count() - n0
        return self.loss_buf

    @property
    def launches_per_step(self):
        """kernels of libt2b200 per optimisation step (graph replays re-launch the captured ones)"""
        return getattr(self, "_fwd_bwd_launches", 0) + getattr(self, "_opt_launches", 0)

    def time_kernel(self, which, layer, reps=20):
        """which: 0 gate GEMM, 1 out GEMM, 2 dz/gate-backward GEMM, 3 dx GEMM -> average ms per launch"""
        ms = ctypes.c_float()
        L.check(self.lib.t2_wn_time_kernel(ctypes.byref(self.cfg), L.ptr(self.params), L.ptr(self.packed),
                                           L.ptr(self.workspace), which, layer, reps, ctypes.byref(ms), L.stream_ptr()))
        return ms.value

    def time_gate_gemm(self, layer, reps=20):
        return self.time_kernel(0, layer, reps)

    def learning_rate(self):
        hp = self.hp
        if hp.wavenet_lr_schedule == "noam":
            step = float(self.global_step + 1)
            w = hp.wavenet_warmup
            return max(hp.wavenet_learning_rate * w ** 0.5 * min(step * w ** -1.5, step ** -0.5), 1e-4)
        return hp.wavenet_learning_rate * hp.wavenet_decay_rate ** (self.global_step / hp.wavenet_decay_steps)

    def optimizer_step(self, grad_scale=1.0):
        """Adam + per-tensor clip (wavenet.py:586-593) + EMA (:613) on the flat buffers."""
        hp = self.hp
        if self.m is None:
            self.m = torch.zeros_like(self.params)
            self.v = torch.zeros_like(self.params)
            self.ema = self.params.clone()
        lr = self.learning_rate()
        clip = hp.wavenet_clip_gradients
        L.check(self.lib.t2_adam_step(
            L.ptr(self.params), L.ptr(self.grads), L.ptr(self.m), L.ptr(self.v), L.ptr(self.ema),
            L.ptr(self.offsets), len(self.tensors), ctypes.c_longlong(self.n_params), ctypes.c_float(lr),
            ctypes.c_float(hp.wavenet_adam_beta1), ctypes.c_float(hp.wavenet_adam_beta2),
            ctypes.c_float(hp.wavenet_adam_epsilon), self.global_step + 1, ctypes.c_float(grad_scale),
            ctypes.c_float(hp.wavenet_gradient_max_norm if clip else 0.0),
            ctypes.c_float(hp.wavenet_gradient_max_value if clip else 0.0), ctypes.c_float(0.0),
            ctypes.c_float(hp.wavenet_ema_decay), L.ptr(self.opt_scratch), L.stream_ptr()))
        self.global_step += 1
        self._packed_dirty = True
        return lr

    def workspace_tensor(self, name, shape=None):
        p = ctypes.c_void_p()
        cnt = ctypes.c_longlong()
        eb = ctypes.c_int()
        L.check(self.lib.t2_wn_workspace_tensor(ctypes.byref(self.cfg), L.ptr(self.workspace), name.encode(),
                                                ctypes.byref(p), ctypes.byref(cnt), ctypes.byref(eb)))
        off = p.value - self.workspace.data_ptr()
        raw = self.workspace[off:off + cnt.value * eb.value]
        t = raw.view(torch.bfloat16 if eb.value == 2 else torch.float32)
        return t.reshape(shape) if shape is not None else t

    def loss_value(self):
        s, n = self.loss_buf.tolist()
        if self.chain_errors():
            raise RuntimeError("a persistent layer-chain launch timed out waiting for a tile and skipped the rest of its work")
        return s / max(n, 1e-20)

    def chain_errors(self):
        """Launches of the persistent layer chains (t2_wn_forward / backward) whose dependency waits timed out since t2_wn_init."""
        p, n, eb = ctypes.c_void_p(), ctypes.c_longlong(), ctypes.c_int()
        L.check(self.lib.t2_wn_workspace_tensor(ctypes.byref(self.cfg), L.ptr(self.workspace), b"chain_err", ctypes.byref(p),
                                                ctypes.byref(n), ctypes.byref(eb)))
        off = p.value - self.workspace.data_ptr()
        return int(self.workspace[off:off + 4].view(torch.int32).item())


class WaveNetSynthesizer(object):
    """Fast-WaveNet autoregressive generation on the H100 (wavenet_vocoder/synthesizer.py + WaveNet.incremental)."""

    def __init__(self, hparams, B, T, cluster_size=8, device="cuda", precision="bf16"):
        """precision: 'bf16' (synthesis weights and conditioning stored in bf16, fp32 arithmetic) or 'fp32-class' (fp32 weights and
        conditioning: the raw outputs differ from the fp32 network only by fp32 accumulation order)."""
        self.hp = hparams
        self.lib = L.load()
        self.device = torch.device(device)
        self.precision = precision
        self.cfg = make_config(hparams, B, T, False, 0.0, precision)
        self.cs = cluster_size
        sz = WnSizes()
        L.check(self.lib.t2_wn_sizes(ctypes.byref(self.cfg), ctypes.byref(sz)))
        self.n_params = sz.n_params
        self.params = torch.zeros(sz.n_params, dtype=torch.float32, device=self.device)
        pb, wb = ctypes.c_longlong(), ctypes.c_longlong()
        L.check(self.lib.t2_wn_ar_sizes(ctypes.byref(self.cfg), self.cs, ctypes.byref(pb), ctypes.byref(wb)))
        self.packed = torch.empty(pb.value, dtype=torch.uint8, device=self.device)
        self.workspace = torch.zeros(wb.value, dtype=torch.uint8, device=self.device)
        self._spk = torch.zeros(B, dtype=torch.int32, device=self.device) if self.cfg.gin_channels > 0 else None
        self.tensors = L.param_table(self.lib.t2_wn_param_info, self.cfg, sz.n_tensors, trainable=False)

    def load_params(self, params):
        flat = torch.zeros(self.n_params, dtype=torch.float32)
        for name, off, shape in self.tensors:
            flat[off:off + int(math.prod(shape))] = params[name].detach().float().reshape(-1)
        self.params.copy_(flat.to(self.device))
        L.check(self.lib.t2_wn_ar_pack(ctypes.byref(self.cfg), self.cs, L.ptr(self.params), L.ptr(self.packed),
                                       L.ptr(self.workspace), L.stream_ptr()))

    def init_variables(self, seed=None):
        from . import init
        self.load_params(init.wavenet_variables(self.hp, self.tensors, seed))

    def generate(self, c, initial, test_inputs=None, u_a=None, u_b=None, seed=0, return_raw=False, speakers=None):
        """c: fp32 [B,cin,Tc]; initial: int32/fp32 [B]; speakers: ids [B] / [B, 1] (gin_channels > 0; None = no speaker term).
        Returns samples [B,T] (and raw outputs [B,T,out])."""
        B, T = self.cfg.B, self.cfg.T
        if speakers is not None and self._spk is None:
            raise L.T2Error("speaker ids need gin_channels > 0")
        if self._spk is not None:
            if speakers is not None:
                self._spk.copy_(speaker_ids(speakers, B, self.cfg.n_speakers))
            L.check(self.lib.t2_wn_ar_set_speakers(ctypes.byref(self.cfg), self.cs, L.ptr(self.params), L.ptr(self.packed),
                                                   L.ptr(self.workspace), None if speakers is None else L.ptr(self._spk),
                                                   L.stream_ptr()))
        if self.hp.upsample_type == "NearestNeighbor" and c is not None and c.dim() == 3 and c.shape[1] == self.cfg.cin_channels and c.shape[2] != T:
            c = nn_upsample(self.hp, c, T)
        scalar = self.cfg.input_type != 2
        out = torch.empty(B, T, dtype=torch.float32 if scalar else torch.int32, device=self.device)
        raw = torch.empty(B, T, self.cfg.out_channels, dtype=torch.float32, device=self.device) if return_raw else None
        L.check(self.lib.t2_wn_ar_generate(ctypes.byref(self.cfg), self.cs, L.ptr(self.params), L.ptr(self.packed),
                                           L.ptr(self.workspace), L.ptr(c), L.ptr(initial), L.ptr(test_inputs),
                                           L.ptr(u_a), L.ptr(u_b), ctypes.c_ulonglong(seed), L.ptr(out), L.ptr(raw),
                                           L.stream_ptr()))
        return (out, raw) if return_raw else out
