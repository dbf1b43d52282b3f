"""Decode-time runtime helpers around QuantLinearLUT (public API).

`GraphedDecodeStep` turns a token step made of QuantLinearLUT calls (224 of them per LLaMA-7B token, each a
short kernel) into ONE CUDA-graph replay with static device buffers and pinned host staging:

    runner = GraphedDecodeStep(step_fn, example_x)      # captures step_fn(x_dev) -> y_dev
    y_host = runner(x_host)                             # H2D copy, replay, D2H copy, all on one stream

It exists because the reference drives the path from Python one launch at a time on the legacy stream
(llama.py:226-234, quant_cuda_kernel.cu:147), which costs more host time per call than the kernels take on an
H100; our kernels launch on the current stream precisely so that they can be captured.
"""
import itertools
import math
import numbers
from typing import NamedTuple

import torch


class GraphedDecodeStep:
    """A decode step captured once as a CUDA graph and replayed; an inference path: its outputs carry no gradient."""

    def __init__(self, step_fn, example_x, warmup=3, static_input=False):
        """static_input=True: `example_x` itself is the static input buffer (a DecodeSequence's `x`), not a clone of it."""
        assert example_x.is_cuda, "example_x must be a CUDA tensor (static input buffer is cloned from it)"
        self.step_fn = step_fn
        self.x_dev = example_x if static_input else example_x.clone()
        self.x_host = torch.empty(example_x.shape, dtype=example_x.dtype, pin_memory=True)
        self.stream = torch.cuda.Stream()
        self.stream.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(self.stream):
            for _ in range(warmup):  # also sizes the per-stream fused-path workspace before capture
                y = step_fn(self.x_dev)
        torch.cuda.current_stream().wait_stream(self.stream)
        torch.cuda.synchronize()
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph, stream=self.stream):
            self.y_dev = step_fn(self.x_dev)
        self.y_host = torch.empty(self.y_dev.shape, dtype=self.y_dev.dtype, pin_memory=True)
        self.h2d_bytes = self.x_host.numel() * self.x_host.element_size()
        self.d2h_bytes = self.y_host.numel() * self.y_host.element_size()

    def replay(self):
        """Device-only: replay on the current stream with whatever is in the static input buffer."""
        self.graph.replay()
        return self.y_dev

    def __call__(self, x_host):
        """End to end from host memory: pinned H2D, replay, pinned D2H, synchronise; returns the pinned host result."""
        self.x_host.copy_(x_host)
        self.x_dev.copy_(self.x_host, non_blocking=True)
        self.graph.replay()
        self.y_host.copy_(self.y_dev, non_blocking=True)
        torch.cuda.current_stream().synchronize()
        return self.y_host


class SeqVec:
    """A vector inside a DecodeSequence: an external input (item -1: `seq.x`; -2, -3, ...: the vectors of `new_input`) or (a slice of)
    the output of one of its matvecs."""

    def __init__(self, item, offset, length):
        self.item, self.offset, self.length = item, offset, length

    def __getitem__(self, sl):
        assert isinstance(sl, slice) and sl.step in (None, 1), "SeqVec supports contiguous slices only"
        a, b, _ = sl.indices(self.length)
        return SeqVec(self.item, self.offset + a, max(0, b - a))

    def __len__(self):
        return self.length


class DecodeSequence:
    """A token step recorded as a list of dependent QuantLinearLUT matvecs and run as ONE persistent kernel launch
    (csrc/lutgemv_seq.cuh): the weight stream never stops between two matvecs and results travel from one matvec to the
    next as self-validating tagged words - no launch, no grid barrier in between.  An inference path: its results carry no
    gradient.

        seq = DecodeSequence(hidden, device)                  # seq.x: static input buffer [hidden] (fp16, or dtype=torch.bfloat16)
        qkv = seq.matvec(stacked_qkv_layer, seq.input)        # -> SeqVec over the full output
        o   = seq.matvec(o_proj, qkv[2 * hidden:3 * hidden])
        ...
        seq.compile(outputs=[d])                              # d: the SeqVec whose plain copy is wanted
        y = seq.replay()[0]                                   # run on the current stream (CUDA-graph capturable)

    It replaces the per-layer launch loop of the reference's decode (llama.py:226-234) for the QuantLinear layers; whatever
    sits between them in a real model (attention, norms) has to run as its own launches, i.e. a model is cut into sequences
    at those points.  Layers must be QuantLinearLUT modules of one bit width, on one device.
    `dtype` is the activation type, torch.float16 or torch.bfloat16: that of `x`, of the values handed from one matvec to the next
    and of the outputs; every output is rounded to it once, with the bias inside the fp32 sum.  A bf16 sequence uses the exact
    codebook whatever `lut_mode` says (the fp16 pair table multiplies fp16 by fp16), as QuantLinearLUT does for one bf16 row.
    On several GPUs pass `peer` (sharding.PeerArena): every layer is this rank's column shard.

    What a decoder layer puts between two matvecs runs inside the same launch (`matvec`'s keywords): an RMSNorm of the input, SiLU
    gating of the input by a second vector, a residual added to the output - each rounded to `dtype` once (lutgemv_seq.cuh)."""

    def __init__(self, in_features, device, lut_mode=None, peer=None, dtype=torch.float16, x=None):
        """x: a tensor the sequence reads as its input instead of a buffer of its own (another kernel's output, say), not copied."""
        if dtype not in (torch.float16, torch.bfloat16):
            raise ValueError(f"DecodeSequence: dtype must be torch.float16 or torch.bfloat16 (got {dtype})")
        self.device = torch.device(device)
        self.dtype = dtype
        self.x = self._bind(x, in_features, "x")
        self.input = SeqVec(-1, 0, in_features)
        self._ext = [self.x]   # external vector of item -1 - j: self._ext[j]
        self._items, self._lens, self._keep, self._ops = [], [], [], []
        self._handle, self.outputs, self._out_vecs = None, [], []
        self.lut_mode = lut_mode
        self.peer = peer

    def _bind(self, t, n, name):
        """A new zero vector of n elements, or the checked tensor t that the sequence reads in its place."""
        if t is None:
            return torch.zeros(n, dtype=self.dtype, device=self.device)
        if not isinstance(t, torch.Tensor):
            raise TypeError(f"DecodeSequence: {name} must be a tensor (got {type(t).__name__})")
        if t.dtype != self.dtype:
            raise ValueError(f"DecodeSequence: {name} has dtype {t.dtype}, the sequence's is {self.dtype}")
        dev = self.device
        if dev.type == "cuda" and dev.index is None:
            dev = torch.device("cuda", torch.cuda.current_device())
        if t.device != dev:
            raise ValueError(f"DecodeSequence: {name} is on {t.device}, the sequence on {self.device}")
        if t.dim() != 1 or t.numel() != n or not t.is_contiguous():
            raise ValueError(f"DecodeSequence: {name} must be a contiguous vector of {n} elements (got shape {tuple(t.shape)})")
        if t.data_ptr() % 16:
            raise ValueError(f"DecodeSequence: {name} must be 16-byte aligned")
        return t

    def new_input(self, n, tensor=None):
        """Another external vector of n elements: (its SeqVec, its static tensor), read by every run like `x`.  tensor: read this one
        (another sequence's output, say) instead of a new buffer, not copied."""
        assert self._handle is None, "sequence already compiled"
        t = self._bind(tensor, n, "tensor")
        self._ext.append(t)
        return SeqVec(-len(self._ext), 0, n), t

    def _ext_tensor(self, v):
        t = self._ext[-v.item - 1]
        return t if v.offset == 0 and v.length == t.numel() else t[v.offset:v.offset + v.length]

    def matvec(self, layer, x, members=1, *, norm=None, up=None, residual=None):
        """Record y = layer(x).  `members`: on several GPUs, how many equal column shards `layer` stacks (q/k/v: 3).
        norm=(weight, eps): the layer reads RMSNorm(x) (weight [in_features] of the sequence's dtype); up=SeqVec: it reads
        silu(x) * up (up: an earlier matvec's output); residual=SeqVec: y = layer(...) + residual, the residual of y's full length."""
        assert self._handle is None, "sequence already compiled"
        assert isinstance(x, SeqVec) and x.length == layer.infeatures, f"input has {len(x)} elements, layer wants {layer.infeatures}"
        assert x.item < len(self._items)
        assert norm is None or up is None, "one input transform per matvec: norm or up"
        world = self.peer.world if self.peer is not None else 1
        assert layer.outfeatures % members == 0
        nfull = layer.outfeatures // members * world
        rows, cols, vals, fr, fri = layer._sparse_args()
        self._items.append((layer.qweight, layer.lookup_table, layer.bits, layer.bias, rows, cols, vals, fr, fri,
                            x.item, x.offset, self._ext_tensor(x) if x.item < 0 else None, members, nfull))
        self._keep.append(layer)
        self._lens.append(members * nfull)
        op = None
        if norm is not None or up is not None or residual is not None:
            x_op, weight, eps, x2 = 0, None, 0.0, (-1, 0)
            if norm is not None:
                weight, eps = norm
                assert weight.numel() == layer.infeatures, f"norm weight has {weight.numel()} elements, layer wants {layer.infeatures}"
                x_op, weight = 1, weight.to(device=self.device, dtype=self.dtype).contiguous()
                self._keep.append(weight)
            if up is not None:
                assert isinstance(up, SeqVec) and 0 <= up.item < len(self._items) - 1, "up must be an earlier matvec's output"
                assert up.length == layer.infeatures, f"up has {len(up)} elements, layer wants {layer.infeatures}"
                x_op, x2 = 2, (up.item, up.offset)
            res, res_ext = (-1, 0), None
            if residual is not None:
                assert isinstance(residual, SeqVec) and residual.length == members * nfull, \
                    f"residual has {len(residual)} elements, the output has {members * nfull}"
                if residual.item >= 0:
                    res = (residual.item, residual.offset)
                else:
                    res_ext = self._ext_tensor(residual)
            op = (x_op, weight, float(eps), x2[0], x2[1], res[0], res[1], res_ext)
        self._ops.append(op)
        return SeqVec(len(self._items) - 1, 0, members * nfull)

    def compile(self, outputs):
        from .quant import quant_cuda
        assert self._handle is None and self._items
        mode = self.lut_mode or quant_cuda.get_lut_mode()
        exports, bufs = [], {}
        for v in outputs:
            assert v.item >= 0, "the input is not an output"
            if v.item not in bufs:
                bufs[v.item] = torch.zeros(self._lens[v.item], dtype=self.dtype, device=self.device)
                exports.append((v.item, bufs[v.item]))
        self.outputs = [bufs[v.item][v.offset:v.offset + v.length] for v in outputs]
        ops = self._ops if any(o is not None for o in self._ops) else None
        with torch.cuda.device(self.device):
            if self.peer is not None:
                arena, peer_base = self.peer.arena_for(quant_cuda.sequence_arena_bytes(self._lens))
                self._handle = quant_cuda.sequence_create(self._items, exports, mode, self.peer.world, self.peer.rank, arena, peer_base,
                                                          dtype=self.dtype, ops=ops)
                self._arena = arena
            else:
                self._handle = quant_cuda.sequence_create(self._items, exports, mode, dtype=self.dtype, ops=ops)
        self._exports = exports
        self._quant_cuda = quant_cuda
        return self

    def replay(self):
        """Run on the current stream with whatever is in `self.x`; returns the output views (static buffers)."""
        self._quant_cuda.sequence_run(self._handle)
        return self.outputs

    def error(self):
        """True if a bounded in-kernel wait (2 s) ever gave up: a result since then is incomplete.  Synchronises the current stream."""
        return self._quant_cuda.sequence_error(self._handle)

    def check(self):
        if self.error():
            raise RuntimeError("DecodeSequence: an in-kernel wait timed out (2 s) - on several GPUs a rank was late or absent; results since then "
                               "are incomplete.  Bring the ranks together (barrier) and call reset_error() on every rank.")

    def reset_error(self):
        self._quant_cuda.sequence_reset_error(self._handle)

    def __del__(self):
        try:
            if self._handle is not None:
                self._quant_cuda.sequence_destroy(self._handle)
                self._handle = None
        except Exception:
            pass


# ---- whole-model greedy decode -----------------------------------------------------------------------------------------------------
DECODER_CLASSES = ("LlamaForCausalLM", "MistralForCausalLM", "Qwen2ForCausalLM")
_PROJ = (("self_attn", ("q_proj", "k_proj", "v_proj", "o_proj")), ("mlp", ("gate_proj", "up_proj", "down_proj")))


class PlanItem(NamedTuple):
    """One matvec of a decoder sequence.  x / up / residual are (source, offset, length): source "x" is the sequence's input, "h" its
    residual input, anything else the output of an earlier item of the same sequence.  norm is the RMSNorm module whose weight and eps
    the item applies to its input."""
    name: str
    layer: object
    x: tuple
    norm: object = None
    up: tuple = None
    residual: tuple = None


class SeqPlan(NamedTuple):
    """One DecodeSequence: its input ("embed": the token's embedding, "attn": the attention output), its residual input h (None, "embed"
    or (sequence name, item name): an exported output of an earlier sequence), its items and the item outputs it exports."""
    name: str
    x: str
    h: object
    items: list
    outputs: list


class AttnPlan(NamedTuple):
    """The attention launch of decoder layer `layer`, reading the stacked q|k|v output (sequence name, item name)."""
    layer: int
    qkv: tuple


def _decoder_layout(model, max_len, who="SequenceDecoder"):
    """The checks of SequenceDecoder (and BatchDecoder: `who`) that need no device, in the order they are made; raises ValueError
    naming the reason.  Returns the model's decoder layers."""
    import transformers
    name = type(model).__name__
    if name not in DECODER_CLASSES or type(model) is not getattr(transformers, name):
        raise ValueError(f"{who}: {name} is not supported (only {', '.join(DECODER_CLASSES)})")
    if not isinstance(max_len, int) or max_len < 1:
        raise ValueError(f"{who}: max_len must be a positive int (got {max_len!r})")
    cfg = model.config
    if "sliding_attention" in (getattr(cfg, "layer_types", None) or ()):
        raise ValueError(f"{who}: sliding-window attention is not supported (config.layer_types has sliding_attention layers)")
    if name == "MistralForCausalLM" and cfg.sliding_window is not None and cfg.sliding_window < max_len:
        raise ValueError(f"{who}: sliding-window attention is not supported (sliding_window={cfg.sliding_window} < "
                         f"max_len={max_len})")
    if getattr(cfg, "hidden_act", "silu") != "silu":
        raise ValueError(f"{who}: hidden_act={cfg.hidden_act!r} is not silu")
    layers = model.model.layers
    head_dim = layers[0].self_attn.head_dim
    if head_dim not in (64, 128):
        raise ValueError(f"{who}: head_dim={head_dim} is not 64 or 128")
    from .quant import QuantLinearLUT
    quant = []
    for i, layer in enumerate(layers):
        for block, names in _PROJ:
            for n in names:
                m = getattr(getattr(layer, block), n)
                if not isinstance(m, QuantLinearLUT):
                    raise ValueError(f"{who}: layers.{i}.{block}.{n} is a {type(m).__name__}, not a QuantLinearLUT")
                quant.append((f"layers.{i}.{block}.{n}", m))
    if isinstance(model.lm_head, QuantLinearLUT):
        quant.append(("lm_head", model.lm_head))
    bits = sorted({m.bits for _, m in quant})
    if len(bits) > 1:
        raise ValueError(f"{who}: mixed bit widths {bits}: the layers must share one")
    for n, m in quant:
        if m._trained:
            raise ValueError(f"{who}: {n} is being trained (train_codebook: {', '.join(m._trained)})")
    dtype = model.model.embed_tokens.weight.dtype
    if dtype not in (torch.float16, torch.bfloat16):
        raise ValueError(f"{who}: the model is {dtype}; only float16 and bfloat16 models are supported")
    return layers


def _check_rows_fit(model, layers, who):
    """ValueError naming the first projection of a multi-row step (stacked q/k/v, o, stacked gate/up, down and a quantized lm_head)
    that does not fit the multi-row LUT-GEMV (QuantLinearLUT._rows_fits); the shapes are those of the stacked siblings, checked before
    anything is stacked."""
    import types

    from .quant import FUSED_LIMITS, QuantLinearLUT
    for i, layer in enumerate(layers):
        at, mlp = layer.self_attn, layer.mlp
        shapes = [("self_attn.q_proj|k_proj|v_proj", at.q_proj.infeatures,
                   at.q_proj.outfeatures + at.k_proj.outfeatures + at.v_proj.outfeatures),
                  ("self_attn.o_proj", at.o_proj.infeatures, at.o_proj.outfeatures),
                  ("mlp.gate_proj|up_proj", mlp.gate_proj.infeatures, mlp.gate_proj.outfeatures + mlp.up_proj.outfeatures),
                  ("mlp.down_proj", mlp.down_proj.infeatures, mlp.down_proj.outfeatures)]
        if i == len(layers) - 1 and isinstance(model.lm_head, QuantLinearLUT):
            shapes.append(("lm_head", model.lm_head.infeatures, model.lm_head.outfeatures))
        for n, K, N in shapes:
            if not QuantLinearLUT._rows_fits(types.SimpleNamespace(infeatures=K, outfeatures=N)):
                where = n if n == "lm_head" else f"layers.{i}.{n}"
                raise ValueError(f"{who}: {where} ({K} -> {N}) does not fit the multi-row LUT-GEMV (out_features a multiple "
                                 f"of 4, in_features up to {FUSED_LIMITS['rows_max_in_features']})")


def _stacked(module, names, who):
    """The stacked layer of the sibling group that holds exactly module.<names>, in that order."""
    ms = [getattr(module, n) for n in names]
    g = ms[0]._sibling_group
    if g is None or g[0].members != ms:
        raise ValueError(f"{who}: {', '.join(names)} are not one sibling group (fusion.fuse_siblings could not stack them)")
    return g[0].layer


def _model_device(model, who):
    """The one GPU every tensor of the model is on; ValueError otherwise."""
    devs = {p.device for p in model.parameters()} | {b.device for b in model.buffers()}
    if len(devs) != 1 or next(iter(devs)).type != "cuda":
        raise ValueError(f"{who}: the model must be on one GPU (its tensors are on {sorted(map(str, devs))})")
    return next(iter(devs))


def _rope_tables(model, max_len, head_dim, device):
    """fp32 cos, sin [max_len, head_dim/2] of the model's own rotary embedding at positions 0 .. max_len-1 (any rope type)."""
    cos, sin = model.model.rotary_emb(torch.zeros(1, dtype=torch.float32, device=device), torch.arange(max_len, device=device)[None])
    return cos[0, :, :head_dim // 2].float().contiguous(), sin[0, :, :head_dim // 2].float().contiguous()


def decoder_plan(model, max_len):
    """What SequenceDecoder runs for one token, in order: SeqPlan and AttnPlan entries.  Stacks the model's siblings
    (fusion.fuse_siblings), which leaves its outputs as they were.  A prologue sequence qkv_0 = qkv(rmsnorm(embed)); per layer l its
    attention, then one sequence o = o_proj(attn) + h, gu = gate_up(rmsnorm(o)), d = down(silu(g) u) + o and qkv_{l+1} = qkv(rmsnorm(d)),
    the last layer's ending in lm_head(rmsnorm(d)) instead when lm_head is a QuantLinearLUT (else the final norm and lm_head run as
    torch ops on its d)."""
    layers = _decoder_layout(model, max_len)
    return _plan(model, layers, *_stack_siblings(model, layers, "SequenceDecoder"))


def _stack_siblings(model, layers, who):
    """fusion.fuse_siblings(model), then the stacked q/k/v layers and the stacked gate/up layers of the decoder layers."""
    from .fusion import fuse_siblings
    fuse_siblings(model)
    return ([_stacked(layer.self_attn, _PROJ[0][1][:3], who) for layer in layers],
            [_stacked(layer.mlp, _PROJ[1][1][:2], who) for layer in layers])


def _plan(model, layers, qkv, gate_up):
    """decoder_plan's list from the decoder layers and their stacked q/k/v and gate/up layers."""
    from .quant import QuantLinearLUT
    H = model.config.hidden_size
    plan = [SeqPlan("prologue", "embed", None, [PlanItem("qkv", qkv[0], ("x", 0, H), layers[0].input_layernorm)], ["qkv"])]
    for i, layer in enumerate(layers):
        prev = plan[-1].name
        plan.append(AttnPlan(i, (prev, "qkv")))
        I = layer.mlp.down_proj.infeatures
        o_proj = layer.self_attn.o_proj
        items = [PlanItem("o", o_proj, ("x", 0, o_proj.infeatures), residual=("h", 0, H)),
                 PlanItem("gu", gate_up[i], ("o", 0, H), layer.post_attention_layernorm),
                 PlanItem("d", layer.mlp.down_proj, ("gu", 0, I), up=("gu", I, I), residual=("o", 0, H))]
        if i + 1 < len(layers):
            items.append(PlanItem("qkv", qkv[i + 1], ("d", 0, H), layers[i + 1].input_layernorm))
            outputs = ["d", "qkv"]
        elif isinstance(model.lm_head, QuantLinearLUT):
            items.append(PlanItem("logits", model.lm_head, ("d", 0, H), model.model.norm))
            outputs = ["logits"]
        else:
            outputs = ["d"]
        plan.append(SeqPlan(f"layer{i}", "attn", "embed" if i == 0 else (prev, "d"), items, outputs))
    return plan


def _sampling(who, n, temperature, top_k, top_p, seed):
    """generate's sampling keywords as four lists of n values, one per prompt (temperature, top_k, top_p, seed), or None when every
    temperature is 0 (greedy: generate then launches no sampler).  A scalar applies to every prompt, except a scalar seed s, which gives
    prompt i the seed s + i, so that identical prompts of one call do not draw alike.  Raises ValueError, before anything runs, for a
    temperature that is negative or not finite, a top_k that is not an int >= 0, a top_p outside (0, 1], a seed outside [0, 2^63) or a
    list whose length is not n."""
    def per_prompt(name, v):
        if isinstance(v, (list, tuple)):
            if len(v) != n:
                raise ValueError(f"{who}: {name} has {len(v)} values for {n} prompt(s)")
            return list(v)
        return None

    def real(v):
        return isinstance(v, numbers.Real) and not isinstance(v, bool)

    def integer(v):
        return isinstance(v, numbers.Integral) and not isinstance(v, bool)

    temps = per_prompt("temperature", temperature) or [temperature] * n
    ks = per_prompt("top_k", top_k) or [top_k] * n
    ps = per_prompt("top_p", top_p) or [top_p] * n
    seeds = per_prompt("seed", seed) or ([seed + i for i in range(n)] if integer(seed) else [seed] * n)
    for t in temps:
        if not real(t) or not math.isfinite(t) or t < 0:
            raise ValueError(f"{who}: temperature must be a finite number >= 0 (got {t!r})")
    for k in ks:
        if not integer(k) or k < 0:
            raise ValueError(f"{who}: top_k must be an int >= 0 (got {k!r})")
    for p in ps:
        if not real(p) or not 0 < p <= 1:
            raise ValueError(f"{who}: top_p must be a number in (0, 1] (got {p!r})")
    for s in seeds:
        if not integer(s) or not 0 <= s < 2**63:
            raise ValueError(f"{who}: seed must be an int in [0, 2^63) (got {s!r})")
    if all(t == 0 for t in temps):
        return None
    return [float(t) for t in temps], [min(int(k), 2**31 - 1) for k in ks], [float(p) for p in ps], [int(s) for s in seeds]


def _eos_set(eos_token_id):
    """generate's eos_token_id (None, an int or a list of ints) as a set of ints."""
    if eos_token_id is None:
        return set()
    return {int(e) for e in (eos_token_id if isinstance(eos_token_id, (list, tuple)) else [eos_token_id])}


class PromptLookup:
    """The built-in drafter of speculative generate: propose the tokens that followed the most recent earlier occurrence of the last
    n tokens of the history, n = 3 first, then n = 2 (prompt-lookup decoding).  An n-gram -> the index after its last earlier
    occurrence map is kept up to date as tokens arrive, so extend() and propose() cost O(n + k) on the host, not a scan."""

    NGRAMS = (3, 2)

    def __init__(self, tokens=(), k=1):
        self.k = k
        self.tokens = []
        self._after = {}  # n-gram (tuple) -> index of the token after its most recent occurrence that has a token after it
        self.extend(tokens)

    def extend(self, tokens):
        for t in tokens:
            self.tokens.append(int(t))
            i = len(self.tokens) - 1  # the n-grams ending at i - 1 now have a token after them
            for n in self.NGRAMS:
                if i >= n:
                    self._after[tuple(self.tokens[i - n:i])] = i

    def propose(self):
        """Up to k ids (fewer when the occurrence is near the end of the history, none when no suffix n-gram occurred before)."""
        for n in self.NGRAMS:
            if len(self.tokens) > n:
                j = self._after.get(tuple(self.tokens[-n:]))
                if j is not None:
                    return self.tokens[j:j + self.k]
        return []


def accept_length(drafts, draws):
    """The speculative accept rule: the length n of the longest prefix with drafts[i] == draws[i] (draws[i]: the target's own token
    for the position after drafts[i - 1]).  The tokens emitted are draws[0 .. n]."""
    n = 0
    while n < len(drafts) and drafts[n] == draws[n]:
        n += 1
    return n


PAGE = 64  # positions per KV page of a paged decoder: attn::PAGE of the paged attention kernels


class PagePool:
    """The host side of a pool of n_pages KV pages shared by `slots` sequences of up to `width` pages each (no device): the free list,
    each page's reference count and each slot's block table, a list of `width` page ids with -1 where no page is assigned.  A page is
    referenced by every slot whose table names it; it returns to the free list when the last one lets it go.  Every method that can
    fail raises before it changes anything."""

    def __init__(self, n_pages, slots, width):
        self.n_pages, self.width = n_pages, width
        self._free = list(range(n_pages - 1, -1, -1))  # pop() takes the lowest id
        self.refs = [0] * n_pages
        self.tables = [[-1] * width for _ in range(slots)]

    @property
    def free(self):
        """Pages on the free list."""
        return len(self._free)

    def held(self, slot):
        """The number of leading blocks of `slot` that have a page."""
        t = self.tables[slot]
        return next((j for j, x in enumerate(t) if x < 0), len(t))

    def need(self, slot, blocks, fresh=False):
        """Pages assign(slot, blocks, fresh) takes from the free list, net of the pages it gives back."""
        if fresh:
            return blocks - sum(1 for x in self.tables[slot] if x >= 0 and self.refs[x] == 1)
        return max(0, blocks - self.held(slot))

    def assign(self, slot, blocks, fresh=False):
        """Give `slot` pages for its blocks 0 .. blocks-1 (fresh: drop its pages first, so that none of them is shared); RuntimeError
        when the free list is short.  -> [(block, page)] newly assigned."""
        h = 0 if fresh else self.held(slot)
        self.reserve({slot: (blocks, fresh)})
        return [(j, self.tables[slot][j]) for j in range(h, blocks)]

    def reserve(self, want):
        """assign() for several slots at once, {slot: (blocks, fresh)}: all of them or, with RuntimeError naming the slots, none."""
        if sum(max(0, self.need(b, n, f)) for b, (n, f) in want.items()) > len(self._free):
            raise RuntimeError(f"KV page pool: no free page for slot(s) {sorted(want)} ({len(self._free)} of {self.n_pages} pages "
                               f"free); release a slot first")
        for b, (n, f) in want.items():
            if f:
                self.release(b)
            for j in range(self.held(b), n):
                self.tables[b][j] = p = self._free.pop()
                self.refs[p] = 1

    def release(self, slot):
        """Let go of every page of `slot`; its table becomes all -1."""
        t = self.tables[slot]
        for x in t:
            if x >= 0 and self.refs[x] < 1:
                raise ValueError(f"KV page pool: page {x} of slot {slot} is already free")
        for j, x in enumerate(t):
            if x >= 0:
                self.refs[x] -= 1
                if self.refs[x] == 0:
                    self._free.append(x)
                t[j] = -1

    def fork(self, src, dst, pos):
        """dst (holding no page) starts as src at position pos: the full pages of src before pos are shared, the partly filled one
        (pos % PAGE != 0) is replaced by a fresh page.  RuntimeError without a free page for it.  -> (src's page, dst's page) to
        copy, or None at a page boundary."""
        if any(x >= 0 for x in self.tables[dst]):
            raise ValueError(f"KV page pool: slot {dst} already holds pages")
        full, part = divmod(pos, PAGE)
        if part and not self._free:
            raise RuntimeError(f"KV page pool: no free page for the fork into slot {dst} (0 of {self.n_pages} pages free)")
        for j in range(full):
            x = self.tables[src][j]
            self.tables[dst][j] = x
            self.refs[x] += 1
        if not part:
            return None
        self.tables[dst][full] = p = self._free.pop()
        self.refs[p] = 1
        return self.tables[src][full], p


class _DecoderBase:
    """What SequenceDecoder and BatchDecoder share, for `slots` sequences (SequenceDecoder: one): the set-up, the graph capture, the
    prompts (prefill and extend of one slot), the replay with its full-cache check and the generate loop.  Slot b is row b of pos, tok,
    the attention output and the sampling buffers; _pos holds the slots' host positions (-1: idle).  The caches have one of two layouts:
      contiguous (pages=None)  [n_layers, slots, n_kv, max_len, head_dim]: slot b owns block b, max_len positions for its whole life;
      paged (pages=P)          [n_layers, P, n_kv, PAGE, head_dim]: a pool of P pages of PAGE positions (a page id names the same page in
                               every layer), and block_table [slots, ceil(max_len / PAGE)] int32 on the device: position t of slot b is
                               row t % PAGE of page block_table[b, t // PAGE], -1 where no page is assigned.  _pages (a PagePool)
                               holds the host copy; pages are assigned on the host before anything writes their positions.
    A subclass defines _step (one token of every slot on the current stream: what the graph holds) and reset(), and names itself in
    CACHE_FULL."""

    EXTEND_CHUNK = 2048  # extend() runs a prompt in chunks of at most this many tokens: it bounds the activations of one chunk
    CHECK_EVERY = 8      # generate() looks for EOS every this many steps

    def __init__(self, model, max_len, layers, slots, who, pages=None):
        """After the subclass's device-free checks (layers: _decoder_layout's): the one GPU, the head layout and scale, the stacked
        siblings, then on the device the caches, the attention output, the rotary tables, pos, tok and the sampling buffers."""
        from .quant import quant_cuda
        self.device = _model_device(model, who)
        self.model, self.max_len = model, max_len
        self.dtype = model.model.embed_tokens.weight.dtype
        self._qc = quant_cuda
        cfg = model.config
        attn = layers[0].self_attn
        self.n_layers = cfg.num_hidden_layers
        self.n_heads, self.n_kv, self.head_dim = cfg.num_attention_heads, cfg.num_key_value_heads, attn.head_dim
        self.scale = float(getattr(attn, "scaling", self.head_dim ** -0.5))
        self.qkv, self.gate_up = _stack_siblings(model, layers, who)
        dev, d = self.device, self.head_dim
        with torch.cuda.device(dev), torch.no_grad():
            self.pos = torch.zeros(slots, dtype=torch.int32, device=dev)
            self.tok = torch.zeros(slots, dtype=torch.int64, device=dev)
            if pages is None:
                self._k = torch.zeros(self.n_layers, slots, self.n_kv, max_len, d, dtype=self.dtype, device=dev)
                self._pages = None
            else:
                width = -(-max_len // PAGE)
                self._k = torch.zeros(self.n_layers, pages, self.n_kv, PAGE, d, dtype=self.dtype, device=dev)
                self.block_table = torch.full((slots, width), -1, dtype=torch.int32, device=dev)
                self._pages = PagePool(pages, slots, width)
            self._v = torch.zeros_like(self._k)
            self.attn_out = torch.zeros(slots, self.n_heads * d, dtype=self.dtype, device=dev)
            self.rope_cos, self.rope_sin = _rope_tables(model, max_len, d, dev)
            # the device parameters of quant_cuda.sample, one per slot: temperature, top_k, top_p and seed (greedy until generate sets them)
            self.temperature = torch.zeros(slots, dtype=torch.float32, device=dev)
            self.top_k = torch.zeros(slots, dtype=torch.int32, device=dev)
            self.top_p = torch.ones(slots, dtype=torch.float32, device=dev)
            self.seed = torch.zeros(slots, dtype=torch.int64, device=dev)
        self._pos = [0] * slots

    def _capture(self):
        """From reset(): _step once on a side stream (SequenceDecoder's writes position 0, which a prompt overwrites; BatchDecoder's has
        every slot idle and writes nothing), then its capture as the graph, whose logits are self.logits; reset() again."""
        self.reset()
        self.graph, self.logits = self._graph_of(self._step)
        self.reset()

    def _graph_of(self, fn):
        """fn() once on a side stream, then its capture: (the graph, fn's result in the graph's memory)."""
        with torch.cuda.device(self.device), torch.no_grad():
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                fn()
            torch.cuda.current_stream().wait_stream(side)
            torch.cuda.synchronize()
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph, stream=side):
                out = fn()
            torch.cuda.synchronize()
        return graph, out

    def _set_pos(self, slot, p):
        self.pos[slot] = p
        self._pos[slot] = p

    def _reserve(self, want):
        """Paged: pages for {slot: (positions, fresh)} - the slot's positions 0 .. positions-1, fresh: none shared with another slot,
        none kept from before - all or none (RuntimeError naming the slots, nothing changed), and the new entries into block_table.
        Nothing for a contiguous cache."""
        if self._pages is None:
            return
        held = {b: 0 if f else self._pages.held(b) for b, (n, f) in want.items()}
        self._pages.reserve({b: (-(-n // PAGE), f) for b, (n, f) in want.items()})
        for b, (n, f) in want.items():
            t = self._pages.tables[b]
            if f:
                self.block_table[b].fill_(-1)
            for j in range(held[b], -(-n // PAGE)):
                self.block_table[b, j] = t[j]

    def _drop_pages(self, slot):
        """Paged: `slot`'s pages back to the pool and its block_table row to -1."""
        if self._pages is not None and self._pages.held(slot):
            self._pages.release(slot)
            self.block_table[slot].fill_(-1)

    def _set_sampling(self, params):
        """Rows 0 .. n-1 of the sampling buffers from _sampling's lists of n values."""
        for buf, vals in zip((self.temperature, self.top_k, self.top_p, self.seed), params):
            buf[:len(vals)].copy_(torch.tensor(vals, dtype=buf.dtype))

    def _sample(self, logits):
        """tok[b] = quant_cuda.sample of logits row b at pos[b], for the rows of logits; a row whose pos is -1 keeps its token."""
        n = logits.shape[0]
        self._qc.sample(logits, self.pos[:n], self.temperature[:n], self.top_k[:n], self.top_p[:n], self.seed[:n], self.tok[:n])

    def _proj(self, layer, x):
        """layer(x) in the model's dtype (a batch's bias is added in the bias's dtype, fp32 for a checkpoint's bias)."""
        y = layer(x)
        return y if y.dtype == self.dtype else y.to(self.dtype)

    def _layer(self, i, layer, h, attend):
        """Decoder layer i on the rows h [rows, hidden]: input_layernorm, the stacked q/k/v, attend(qkv) -> the attention output
        [rows, n_heads * head_dim], o_proj plus the residual, post_attention_layernorm, the stacked gate/up, silu(g) u, down plus the
        residual."""
        qkv = self._proj(self.qkv[i], layer.input_layernorm(h))
        h = h + self._proj(layer.self_attn.o_proj, attend(qkv))
        gu = self._proj(self.gate_up[i], layer.post_attention_layernorm(h))
        I = gu.shape[1] // 2
        return h + self._proj(layer.mlp.down_proj, torch.nn.functional.silu(gu[:, :I]) * gu[:, I:])

    def _prefill(self, who, slot, input_ids):
        """The prompt [1, T] (or [T]) through the model's own forward, its KV cache copied into `slot`, whose position becomes T; the
        logits of the last position."""
        ids = torch.as_tensor(input_ids).reshape(1, -1).to(self.device)
        T = ids.shape[1]
        if not 1 <= T <= self.max_len:
            raise ValueError(f"{who}: {T} prompt tokens, the cache holds 1 to {self.max_len}")
        self._reserve({slot: (T, True)})
        with torch.no_grad():
            o = self.model(input_ids=ids, use_cache=True)
            for i, layer in enumerate(o.past_key_values.layers):
                if self._pages is None:
                    self._k[i, slot, :, :T].copy_(layer.keys[0])
                    self._v[i, slot, :, :T].copy_(layer.values[0])
                    continue
                for j in range(-(-T // PAGE)):
                    page, n = self._pages.tables[slot][j], min(PAGE, T - j * PAGE)
                    self._k[i, page, :, :n].copy_(layer.keys[0][:, j * PAGE:j * PAGE + n])
                    self._v[i, page, :, :n].copy_(layer.values[0][:, j * PAGE:j * PAGE + n])
        self._set_pos(slot, T)
        return o.logits[0, -1]

    def _extend(self, who, prompts, named=False):
        """The prompts [(slot, input_ids (1-D))], each at its slot's positions start .. start+T-1 (start: its position, 0 for an idle
        slot), through every layer; the slots must be distinct.  A pass takes the next EXTEND_CHUNK tokens of the prompts in the given
        order, so a prompt may span passes; a pass's segments are (slot, its position so far, its tokens in the pass).  A pass of one
        segment attends with quant_cuda.attn_extend (or attn_extend_paged) on the slot's caches, one of several with
        quant_cuda.attn_extend_batch (or attn_extend_batch_paged).  Each slot's position becomes start + T.  -> the logits of each
        prompt's last token [len(prompts), vocab].  ValueError before anything is written when a prompt is empty, not 1-D or does not
        fit (named: the message names the prompt's index); paged, RuntimeError with nothing changed when the pool lacks pages."""
        work = []  # (slot, start, ids)
        for k, (slot, input_ids) in enumerate(prompts):
            what = f"{who}: prompt {k}" if named else who
            start = max(self._pos[slot], 0)
            ids = torch.as_tensor(input_ids)
            if ids.dim() != 1 or ids.numel() == 0:
                raise ValueError(f"{what}: input_ids must be a non-empty 1-D tensor of token ids (got shape {tuple(ids.shape)})")
            if ids.dtype.is_floating_point or ids.dtype.is_complex or ids.dtype == torch.bool:
                raise ValueError(f"{what}: input_ids must hold integer token ids (got {ids.dtype})")
            if start + ids.numel() > self.max_len:
                raise ValueError(f"{what}: {ids.numel()} tokens at position {start} need {start + ids.numel()} cache positions, "
                                 f"max_len is {self.max_len}")
            work.append((slot, start, ids))
        self._reserve({slot: (start + ids.numel(), False) for slot, start, ids in work})
        ids = torch.cat([x.to(device=self.device, dtype=torch.int64) for _, _, x in work])
        ends = list(itertools.accumulate(x.numel() for _, _, x in work))  # prompt k is tokens begins[k] .. ends[k]-1 of ids
        begins = [e - x.numel() for e, (_, _, x) in zip(ends, work)]
        last = [None] * len(work)
        m = self.model.model
        with torch.no_grad():
            for c0 in range(0, ids.numel(), self.EXTEND_CHUNK):
                c1 = min(ids.numel(), c0 + self.EXTEND_CHUNK)
                segs = []  # (prompt, slot, start, tokens) of the pass
                for k, (slot, start, _) in enumerate(work):
                    a, b = max(c0, begins[k]), min(c1, ends[k])
                    if a < b:
                        segs.append((k, slot, start + a - begins[k], b - a))
                out = torch.empty(c1 - c0, self.n_heads * self.head_dim, dtype=self.dtype, device=self.device)
                h = torch.index_select(m.embed_tokens.weight, 0, ids[c0:c1])
                for i, layer in enumerate(m.layers):
                    def attend(qkv, i=i):
                        if len(segs) == 1:
                            _, slot, start, _ = segs[0]
                            if self._pages is None:
                                self._qc.attn_extend(qkv, start, self.rope_cos, self.rope_sin, self._k[i, slot], self._v[i, slot], out,
                                                     self.n_heads, self.n_kv, self.scale)
                            else:
                                self._qc.attn_extend_paged(qkv, start, self.rope_cos, self.rope_sin, self._k[i], self._v[i],
                                                           self.block_table[slot], out, self.n_heads, self.n_kv, self.scale)
                            return out
                        slots, starts, counts = ([s[j] for s in segs] for j in (1, 2, 3))
                        if self._pages is None:
                            self._qc.attn_extend_batch(qkv, slots, starts, counts, self.rope_cos, self.rope_sin, self._k[i], self._v[i],
                                                       out, self.n_heads, self.n_kv, self.scale)
                        else:
                            self._qc.attn_extend_batch_paged(qkv, slots, starts, counts, self.rope_cos, self.rope_sin, self._k[i],
                                                             self._v[i], self.block_table, out, self.n_heads, self.n_kv, self.scale)
                        return out
                    h = self._layer(i, layer, h, attend)
                for k, *_ in segs:
                    if ends[k] <= c1:
                        last[k] = h[ends[k] - 1 - c0:ends[k] - c0]
            logits = self.model.lm_head(m.norm(torch.cat(last)))
        for slot, start, x in work:
            self._set_pos(slot, start + x.numel())
        return logits

    def _replay(self):
        """One step of every active slot; RuntimeError, before it, when an active slot's cache is full or (paged) when the pool has no
        page for an active slot whose position starts a new page."""
        full = [b for b, p in enumerate(self._pos) if p >= self.max_len]
        if full:
            raise RuntimeError(self.CACHE_FULL.format(slots=full, max_len=self.max_len))
        if self._pages is not None:
            self._reserve({b: (p + 1, False) for b, p in enumerate(self._pos) if p >= 0 and self._pages.held(b) <= p // PAGE})
        self.graph.replay()
        self._pos = [p + 1 if p >= 0 else p for p in self._pos]

    def _finished(self, row):
        """generate's row `row` has come to its EOS."""

    def _generate(self, who, prompts, max_new_tokens, eos, sampling):
        """Prompt i (token ids) prefilled into slot i, then steps until every prompt has max_new_tokens new tokens or its first token in
        the set `eos`, looked for every CHECK_EVERY steps, after which _finished(i).  Sampled with _sampling's lists `sampling`, else
        greedy.  -> the new tokens [slots, max_new_tokens] (on the device) and each prompt's count of them."""
        R = len(prompts)
        out = torch.zeros(len(self._pos), max_new_tokens, dtype=torch.int64, device=self.device)
        if sampling:
            self._set_sampling(sampling)
            self._sample(torch.stack([self._prefill(who, i, p) for i, p in enumerate(prompts)]))
            out[:R, 0].copy_(self.tok[:R])
        else:
            for i, p in enumerate(prompts):
                out[i, 0] = self._prefill(who, i, p).argmax()
        self.tok.copy_(out[:, 0])
        length = [None] * R  # new tokens of a finished row
        n, seen = 1, 0
        while True:
            if eos and (n % self.CHECK_EVERY == 0 or n == max_new_tokens):
                got = out[:R, seen:n].tolist()
                for i in range(R):
                    if length[i] is None:
                        hit = next((seen + j for j, t in enumerate(got[i]) if t in eos), None)
                        if hit is not None:
                            length[i] = hit + 1
                            self._finished(i)
                seen = n
                if all(x is not None for x in length):
                    break
            if n == max_new_tokens:
                break
            self._replay()
            if sampling:
                self._sample(self.logits.view(len(self._pos), -1))
            out[:, n].copy_(self.tok)
            n += 1
        return out, [n if x is None else x for x in length]


class SequenceDecoder(_DecoderBase):
    """Batch-1 decode of a whole quantized LLaMA-family model (LlamaForCausalLM, MistralForCausalLM without an active sliding
    window, Qwen2ForCausalLM without sliding window) on one GPU, in fp16 or bf16.  Its q/k/v/o/gate/up/down projections must be
    QuantLinearLUT layers of one bit width (checkpoint.load_quantized / load_checkpoint, then .cuda()); lm_head may be dense or
    QuantLinearLUT.

        dec = SequenceDecoder(model, max_len=2048)
        ids = dec.generate(input_ids, max_new_tokens=128, eos_token_id=tok.eos_token_id)                   # greedy
        ids = dec.generate(input_ids, 128, eos_token_id=tok.eos_token_id, temperature=0.7, top_p=0.9, seed=1)  # sampled

    One token is one CUDA graph replay: the embedding gather from a device token id, the prologue sequence, then per layer the
    attention kernel (quant_cuda.attn_decode: rotary, KV-cache append, attention) and the layer's DecodeSequence (decoder_plan), then
    the final norm and lm_head, the argmax into the device token id and pos += 1.  Tokens follow each other with no host
    synchronisation.  The prompt runs through the model's own forward (prefill), whose cache is copied into the decoder's static one, or
on the decoder's own kernels (extend), which also appends a new turn to the sequence already in the cache.

    Sampling (generate's temperature, top_k, top_p and seed) runs quant_cuda.sample after each replay, on the same stream: it overwrites
    the graph's argmax in tok with a draw keyed by the seed and counted by the position, so tokens still follow each other with no host
    synchronisation.  A step() user samples the same way: quant_cuda.sample(dec.logits.view(1, -1), dec.pos, dec.temperature, dec.top_k,
    dec.top_p, dec.seed, dec.tok) after step() draws the token of position dec.position (fill the four parameter buffers first).

    Speculation (speculate=K in 1..15) adds a second graph, the verify step: T = K + 1 tokens at positions pos .. pos+K in one pass -
    the embedding gather of the device ids, per layer the stacked projections on [T, hidden] (QuantLinearLUT.forward: the multi-row
    kernel, so every projection must fit it) with quant_cuda.attn_verify on the decoder's cache, the final norm, lm_head and the argmax
    of every row.  It reads pos from the device and does not advance it.  generate() then drafts up to K tokens per iteration (the
    built-in PromptLookup, or a `draft` callable), verifies the pending token and the drafts in one replay and keeps the drafts up to the
    first whose target token differs.  Each emitted token is the draw plain generate makes from the same logits at the same position
    (greedy: the argmax; sampled: quant_cuda.sample keyed by the seed and the position), so speculation changes how many positions a
    pass computes, never which token a position gets beyond the rounding of its logits.

    The model itself is changed only by the sibling stacking of fusion.fuse_siblings, which keeps its outputs.  Everything the decoder
    computes carries no gradient."""

    CACHE_FULL = "SequenceDecoder: the cache is full (max_len={max_len}); reset() or prefill() first"

    def __init__(self, model, max_len, speculate=0):
        """speculate: K, the drafted tokens one verify step checks (0: no speculation, no verify graph)."""
        from .quant import QuantLinearLUT
        layers = _decoder_layout(model, max_len)
        if not isinstance(speculate, int) or isinstance(speculate, bool) or not 0 <= speculate <= 15:
            raise ValueError(f"SequenceDecoder: speculate must be an int in 0..15 (got {speculate!r})")
        if speculate:
            _check_rows_fit(model, layers, "SequenceDecoder")
            dtype = model.model.embed_tokens.weight.dtype
            rows_max = QuantLinearLUT.ROWS_MAX if dtype == torch.float16 else QuantLinearLUT.BF16_ROWS_MAX
            if speculate + 1 > rows_max:
                raise ValueError(f"SequenceDecoder: speculate={speculate} needs {speculate + 1} rows, the multi-row LUT-GEMV takes up to "
                                 f"{rows_max} for a {dtype} model")
        super().__init__(model, max_len, layers, 1, "SequenceDecoder")
        # the one slot's views: caches [n_layers, n_kv, max_len, head_dim], attention output [n_heads * head_dim]
        self.k_cache, self.v_cache, self.attn_out = self._k[:, 0], self._v[:, 0], self.attn_out[0]
        self.plan = _plan(model, layers, self.qkv, self.gate_up)
        with torch.cuda.device(self.device), torch.no_grad():
            self._build()
        self._capture()
        self.speculate, self.spec_stats = speculate, None
        if speculate:
            T, dev = speculate + 1, self.device
            with torch.cuda.device(dev), torch.no_grad():
                self.vtok = torch.zeros(T, dtype=torch.int64, device=dev)     # the verify step's ids: pending token, drafts, padding
                self.vdraw = torch.zeros(T, dtype=torch.int64, device=dev)    # row t's token: the argmax, or quant_cuda.sample's draw
                self.vpos = torch.zeros(T, dtype=torch.int32, device=dev)     # row t's sampling position pos + t + 1
                self._vstep = torch.arange(1, T + 1, dtype=torch.int32, device=dev)
                self._vattn = torch.zeros(T, self.n_heads * self.head_dim, dtype=self.dtype, device=dev)
                # quant_cuda.sample's parameters for the T rows (generate copies slot 0's into them)
                self._vsampling = (torch.zeros(T, dtype=torch.float32, device=dev), torch.zeros(T, dtype=torch.int32, device=dev),
                                   torch.ones(T, dtype=torch.float32, device=dev), torch.zeros(T, dtype=torch.int64, device=dev))
            self.reset()
            self.vgraph, self.vlogits = self._graph_of(self._verify_step)
            self.reset()

    def _verify_step(self):
        """The verify step on the current stream: what the verify graph holds.  pos is read, not advanced."""
        m = self.model.model
        h = torch.index_select(m.embed_tokens.weight, 0, self.vtok)
        for i, layer in enumerate(m.layers):
            def attend(qkv, i=i):
                self._qc.attn_verify(qkv, self.pos, self.rope_cos, self.rope_sin, self.k_cache[i], self.v_cache[i], self._vattn,
                                     self.n_heads, self.n_kv, self.scale)
                return self._vattn
            h = self._layer(i, layer, h, attend)
        logits = self.model.lm_head(m.norm(h))
        self.vdraw.copy_(logits.argmax(dim=-1))
        torch.add(self.pos, self._vstep, out=self.vpos)
        return logits

    def _build(self):
        """The DecodeSequences of the plan, each reading its inputs in place: the attention output buffer, the previous sequence's d."""
        self.sequences, self._run, out = [], [], {}
        for step in self.plan:
            if isinstance(step, AttnPlan):
                self._run.append(("attn", step.layer, out[step.qkv]))
                continue
            x = self.attn_out if step.x == "attn" else None
            first = step.items[0]
            seq = DecodeSequence(first.x[2], self.device, dtype=self.dtype, x=x)
            if step.x == "embed":
                out["embed"] = seq.x
            vecs = {"x": seq.input}
            if step.h is not None:
                vecs["h"], _ = seq.new_input(self.model.config.hidden_size, tensor=out[step.h])
            for it in step.items:
                kw = {}
                if it.norm is not None:
                    kw["norm"] = (it.norm.weight.detach(), float(it.norm.variance_epsilon))
                if it.up is not None:
                    kw["up"] = vecs[it.up[0]][it.up[1]:it.up[1] + it.up[2]]
                if it.residual is not None:
                    kw["residual"] = vecs[it.residual[0]][it.residual[1]:it.residual[1] + it.residual[2]]
                vecs[it.name] = seq.matvec(it.layer, vecs[it.x[0]][it.x[1]:it.x[1] + it.x[2]], **kw)
            seq.compile(outputs=[vecs[n] for n in step.outputs])
            for n, t in zip(step.outputs, seq.outputs):
                out[(step.name, n)] = t
            self.sequences.append(seq)
            self._run.append(("seq", seq))
        last = self.plan[-1]
        self._head_in = out[(last.name, last.outputs[0])]
        self._quant_head = last.outputs == ["logits"]

    def _step(self):
        """One token on the current stream: what the graph holds."""
        embed = self.sequences[0].x
        torch.index_select(self.model.model.embed_tokens.weight, 0, self.tok, out=embed.view(1, -1))
        for r in self._run:
            if r[0] == "seq":
                r[1].replay()
            else:
                _, layer, qkv = r
                self._qc.attn_decode(qkv, self.pos, self.rope_cos, self.rope_sin, self.k_cache[layer], self.v_cache[layer],
                                     self.attn_out, self.n_heads, self.n_kv, self.scale)
        if self._quant_head:
            logits = self._head_in
        else:
            logits = self.model.lm_head(self.model.model.norm(self._head_in.view(1, -1)))[0]
        self.tok.copy_(logits.argmax().view(1))
        self.pos.add_(1)
        return logits

    def reset(self):
        """Start a new prompt: position 0 (the cache's old slots are never read again)."""
        self._pos = [0]
        self.pos.zero_()

    @property
    def position(self):
        """The position the next step writes (host copy of the device counter)."""
        return self._pos[0]

    def prefill(self, input_ids):
        """Run the prompt [1, T] (or [T]) through the model's own forward, copy its KV cache into the static one and set the position
        to T; returns the logits of the last position."""
        return self._prefill("SequenceDecoder.prefill", 0, input_ids)

    def extend(self, input_ids):
        """Append the tokens input_ids (1-D) at the current position on the decoder's own kernels (quant_cuda.attn_extend between the
        layers' projections, EXTEND_CHUNK tokens at a time), advance the position by T and return the logits of the last token.  After
        reset() this is a prefill; after prefill(), steps or an earlier extend it continues the sequence (a new turn of a chat, say).
        Raises ValueError, with nothing written, for an empty or non-1-D prompt or one that does not fit in max_len."""
        return self._extend("SequenceDecoder.extend", [(0, input_ids)])[0]

    def step(self, token_id):
        """Feed token_id (an int or a one-element device tensor) at the current position; returns the next-token logits, a static buffer
        that the next step overwrites."""
        if isinstance(token_id, torch.Tensor):
            self.tok.copy_(token_id.reshape(1))
        else:
            self.tok.fill_(int(token_id))
        self._replay()
        return self.logits

    def verify(self, token_ids):
        """Feed the speculate + 1 token ids (ints or a device tensor) at positions p .. p + speculate in one verify replay; returns
        their next-token logits [speculate + 1, vocab], a static buffer that the next verify overwrites, and advances the position by
        speculate + 1 (rewind() takes it back to keep a prefix).  Raises ValueError, with nothing written, on a decoder without
        speculation, for a wrong count or non-integer ids, or when the tokens do not fit in max_len."""
        who = "SequenceDecoder.verify"
        if not self.speculate:
            raise ValueError(f"{who}: the decoder was built with speculate=0; pass speculate=K to SequenceDecoder")
        T = self.speculate + 1
        t = torch.as_tensor(token_ids)
        if t.dtype.is_floating_point or t.dtype.is_complex or t.dtype == torch.bool:
            raise ValueError(f"{who}: token_ids must hold integer token ids (got {t.dtype})")
        if t.numel() != T:
            raise ValueError(f"{who}: {t.numel()} token ids, the verify step takes speculate + 1 = {T}")
        p = self._pos[0]
        if p + T > self.max_len:
            raise ValueError(f"{who}: {T} tokens at position {p} need {p + T} cache positions, max_len is {self.max_len}")
        self.vtok.copy_(t.reshape(T))
        self.vgraph.replay()
        self._set_pos(0, p + T)
        return self.vlogits

    def rewind(self, position):
        """Set the position back to `position` (0 .. the current one): the cache slots from there on are never read again, and the next
        step or verify writes there.  Raises ValueError otherwise."""
        if not isinstance(position, int) or isinstance(position, bool) or not 0 <= position <= self._pos[0]:
            raise ValueError(f"SequenceDecoder.rewind: position must be an int in 0..{self._pos[0]} (got {position!r})")
        self._set_pos(0, position)

    def generate(self, input_ids, max_new_tokens, eos_token_id=None, *, temperature=0.0, top_k=0, top_p=1.0, seed=0, draft=None):
        """input_ids [1, T] followed by up to max_new_tokens tokens, ending after the first EOS (eos_token_id: an int or a list) if one
        comes.  The prompt and max_new_tokens - 1 steps must fit in max_len.  Greedy by default; temperature > 0 samples each token with
        quant_cuda.sample: softmax(logits / temperature), restricted to the top_k largest (0: all) and then to the smallest set of mass
        top_p (1: all), drawn with the random stream of `seed` at the token's position, so a call is reproducible.  Each keyword may also
        be a one-element list.  Bad values raise ValueError before anything runs (see _sampling).

        On a decoder built with speculate=K > 0 generation speculates: `draft` is a callable (the tokens so far, prompt included, as a
        list it must not change) -> a list of proposed next ids, of which the first K are used; None: the built-in PromptLookup.  A
        proposal that is not a list of ints in [0, vocab) raises ValueError.  `draft` on a decoder without speculation raises ValueError.
        spec_stats then holds the call's verify, drafted and accepted counts."""
        who = "SequenceDecoder.generate"
        sampling = _sampling(who, 1, temperature, top_k, top_p, seed)
        if draft is not None and not self.speculate:
            raise ValueError(f"{who}: draft needs a decoder built with speculate > 0")
        if draft is not None and not callable(draft):
            raise ValueError(f"{who}: draft must be a callable (tokens -> list of ids) or None (got {type(draft).__name__})")
        ids = torch.as_tensor(input_ids).reshape(1, -1)
        if max_new_tokens < 1:
            return ids
        if ids.shape[1] + max_new_tokens - 1 > self.max_len:
            raise ValueError(f"SequenceDecoder.generate: {ids.shape[1]} prompt tokens and {max_new_tokens} new ones need "
                             f"{ids.shape[1] + max_new_tokens - 1} cache positions, max_len is {self.max_len}")
        if self.speculate:
            new = self._speculate("SequenceDecoder.prefill", ids, max_new_tokens, _eos_set(eos_token_id), sampling, draft)
            out = torch.tensor([new], dtype=torch.int64, device=self.device)
            n = len(new)
        else:
            out, (n,) = self._generate("SequenceDecoder.prefill", [ids], max_new_tokens, _eos_set(eos_token_id), sampling)
        for seq in self.sequences:
            seq.check()
        return torch.cat([ids.to(self.device), out[:, :n]], dim=1)

    def _speculate(self, who, ids, max_new_tokens, eos, sampling, draft):
        """generate's loop with speculation; -> the new tokens (a list).  One host synchronisation per iteration: the emitted tokens."""
        K, vocab = self.speculate, self.vlogits.shape[-1]
        if sampling:
            self._set_sampling(sampling)
            for buf, vals in zip(self._vsampling, sampling):
                buf.fill_(vals[0])
            self._sample(self._prefill(who, 0, ids).view(1, -1))
            c = int(self.tok)
        else:
            c = int(self._prefill(who, 0, ids).argmax())
        history = [int(t) for t in ids.reshape(-1).tolist()] + [c]
        lookup = PromptLookup(history, K) if draft is None else None
        new = [c]
        self.spec_stats = {"verifies": 0, "drafted": 0, "accepted": 0}
        while len(new) < max_new_tokens and c not in eos:
            p = self._pos[0]
            drafts = lookup.propose() if draft is None else self._check_draft(draft(history), vocab)[:K]
            if not drafts or p + K >= self.max_len:  # one ordinary step, the position advanced by its graph
                self.step(c)
                if sampling:
                    self._sample(self.logits.view(1, -1))
                emitted = [int(self.tok)]
            else:
                m = len(drafts)
                self.vtok.copy_(torch.tensor([c] + drafts + [c] * (K - m), dtype=torch.int64))
                self.vgraph.replay()
                if sampling:
                    self._qc.sample(self.vlogits, self.vpos, *self._vsampling, self.vdraw)
                y = self.vdraw.tolist()
                n = accept_length(drafts, y)
                emitted = y[:n + 1]
                st = self.spec_stats
                st["verifies"], st["drafted"], st["accepted"] = st["verifies"] + 1, st["drafted"] + m, st["accepted"] + n
                for j, t in enumerate(emitted):  # EOS and max_new_tokens cut an accepted run
                    if t in eos or len(new) + j + 1 == max_new_tokens:
                        emitted = emitted[:j + 1]
                        break
                self._set_pos(0, p + len(emitted))  # the fed tokens c, d_1 .. d_j are kept; the rest of the slots is never read
            new += emitted
            history += emitted
            if lookup is not None:
                lookup.extend(emitted)
            c = new[-1]
        return new

    @staticmethod
    def _check_draft(d, vocab):
        """A drafter's proposal as a list of ints in [0, vocab); ValueError otherwise."""
        if isinstance(d, torch.Tensor):
            d = d.tolist()
        if not isinstance(d, (list, tuple)):
            raise ValueError(f"SequenceDecoder.generate: draft must return a list of token ids (got {type(d).__name__})")
        for t in d:
            if not isinstance(t, numbers.Integral) or isinstance(t, bool) or not 0 <= t < vocab:
                raise ValueError(f"SequenceDecoder.generate: draft returned {t!r}, not a token id in [0, {vocab})")
        return [int(t) for t in d]


class BatchDecoder(_DecoderBase):
    """Decode of `batch` sequences at once (2 .. QuantLinearLUT.ROWS_MAX in fp16, 2 .. BF16_ROWS_MAX in bf16) through a whole
    quantized LLaMA-family model on one GPU: the models SequenceDecoder takes, whose projections (stacked q/k/v, o, stacked gate/up,
    down and a quantized lm_head) all fit the multi-row LUT-GEMV (QuantLinearLUT._rows_fits).

        dec = BatchDecoder(model, max_len=2048, batch=8)
        outs = dec.generate([ids_a, ids_b, ids_c], max_new_tokens=128, eos_token_id=tok.eos_token_id)
        outs = dec.generate([ids_a, ids_b], 128, eos_token_id=tok.eos_token_id, temperature=0.7, top_p=0.9, seed=1)

    Each sequence has a slot: row b of every step, its own device position pos[b] and its own cache, so prompts of different lengths need
    no padding and no mask.  The cache has one of two layouts:
      pages=None  block b of k_cache / v_cache [n_layers, batch, n_kv, max_len, head_dim]: every slot holds max_len positions for its
                  whole life, idle or not.
      pages=P     k_cache / v_cache are a pool of P pages of 64 positions, [n_layers, P, n_kv, 64, head_dim], and block_table
                  [batch, ceil(max_len / 64)] (int32, on the device, -1 where no page is assigned) maps slot b's position t to row t % 64
                  of page block_table[b, t // 64].  A slot holds pages for the positions it has used: prefill() and extend() assign
                  the pages of the positions they write, a step assigns one when an active slot's position starts a new page (on the
                  host, before the replay), and release(), reset() and an EOS in generate() give them back; free_pages counts what is
                  left.  When the pool runs dry the call raises RuntimeError naming the slots, with nothing run or changed.  fork(src,
                  dst) starts dst from src's state, sharing src's full pages.  Each row computes the same bits in both layouts.

        dec = BatchDecoder(model, max_len=4096, batch=32, pages=2400)   # 2400 x 64 positions shared by 32 slots  A slot whose pos is -1 is idle: its row still goes
    through the projections, but the attention writes nothing for it, and its logits and token mean nothing.  release() and prefill()
    of a slot between steps while the others keep going is continuous batching.

    One step is one CUDA graph replay: the embedding gather of the device tokens tok[batch]; per layer the model's input_layernorm, the
    stacked q/k/v layer on [batch, hidden] (QuantLinearLUT.forward: the multi-row kernel), quant_cuda.attn_decode_batch on the layer's
    cache, o_proj plus the residual, post_attention_layernorm, the stacked gate/up layer, silu(g) u, down plus the residual; the final
    norm and lm_head, the argmax per row into tok and pos[b] += 1 for the active rows.  Steps follow each other with no host
    synchronisation.  Every op of a step is row-wise, so a row's result does not depend on what the other rows hold.

    Sampling (generate's temperature, top_k, top_p and seed, per prompt) runs quant_cuda.sample after each replay, on the same stream: it
    overwrites the active rows' argmax in tok with draws keyed by each row's seed and counted by its position, so a row's tokens do not
    depend on the other rows either.  A step() user samples the same way: quant_cuda.sample(dec.logits, dec.pos, dec.temperature,
    dec.top_k, dec.top_p, dec.seed, dec.tok) after step() (fill the four [batch] parameter buffers first).

    The model itself is changed only by the sibling stacking of fusion.fuse_siblings, which keeps its outputs.  Everything the decoder
    computes carries no gradient."""

    CACHE_FULL = "BatchDecoder: the cache of slot(s) {slots} is full (max_len={max_len}); release() or prefill() them first"

    def __init__(self, model, max_len, batch, pages=None):
        from .quant import QuantLinearLUT
        layers = _decoder_layout(model, max_len, "BatchDecoder")
        dtype = model.model.embed_tokens.weight.dtype
        rows_max = QuantLinearLUT.ROWS_MAX if dtype == torch.float16 else QuantLinearLUT.BF16_ROWS_MAX
        if not isinstance(batch, int) or not 2 <= batch <= rows_max:
            hint = "; decode one sequence with SequenceDecoder" if batch == 1 else ""
            raise ValueError(f"BatchDecoder: batch must be an int in 2..{rows_max} for a {dtype} model (got {batch!r}){hint}")
        most = batch * -(-max_len // PAGE)
        if pages is not None and (not isinstance(pages, int) or isinstance(pages, bool) or not 1 <= pages <= most):
            raise ValueError(f"BatchDecoder: pages must be None or an int in 1..{most} (batch x ceil(max_len / {PAGE})) (got {pages!r})")
        _check_rows_fit(model, layers, "BatchDecoder")
        super().__init__(model, max_len, layers, batch, "BatchDecoder", pages)
        self.batch = batch
        self.k_cache, self.v_cache = self._k, self._v
        self._capture()

    def _step(self):
        """One step on the current stream: what the graph holds."""
        m = self.model.model
        h = torch.index_select(m.embed_tokens.weight, 0, self.tok)
        for i, layer in enumerate(m.layers):
            def attend(qkv, i=i):
                if self._pages is None:
                    self._qc.attn_decode_batch(qkv, self.pos, self.rope_cos, self.rope_sin, self.k_cache[i], self.v_cache[i],
                                               self.attn_out, self.n_heads, self.n_kv, self.scale)
                else:
                    self._qc.attn_decode_paged(qkv, self.pos, self.rope_cos, self.rope_sin, self.k_cache[i], self.v_cache[i],
                                               self.block_table, self.attn_out, self.n_heads, self.n_kv, self.scale)
                return self.attn_out
            h = self._layer(i, layer, h, attend)
        logits = self.model.lm_head(m.norm(h))
        self.tok.copy_(logits.argmax(dim=-1))
        self.pos.add_((self.pos >= 0).to(torch.int32))
        return logits

    def _slot(self, slot):
        if not isinstance(slot, int) or not 0 <= slot < self.batch:
            raise ValueError(f"BatchDecoder: slot must be an int in 0..{self.batch - 1} (got {slot!r})")
        return slot

    def reset(self):
        """Release every slot."""
        self.pos.fill_(-1)
        self._pos = [-1] * self.batch
        for b in range(self.batch):
            self._drop_pages(b)

    def release(self, slot):
        """Make `slot` idle (pos -1): the steps write nothing for it from now on; its old cache slots are never read again (paged: its
        pages go back to the pool)."""
        self._set_pos(self._slot(slot), -1)
        self._drop_pages(slot)

    _finished = release

    @property
    def free_pages(self):
        """Pages left in the pool (paged), None for the contiguous layout."""
        return None if self._pages is None else self._pages.free

    def fork(self, src, dst):
        """Start idle slot `dst` from active slot `src`'s current state without recomputing it (n samples of one prompt, one system
        prompt under several conversations): dst takes src's position; src's full pages before it are shared (writes only go to
        positions at or past a slot's own, so a shared full page is never written) and its partly filled last page is copied into a
        fresh page in every layer.  Paged decoders only.  ValueError for bad slots, RuntimeError (nothing changed) without a free page
        for the copy."""
        if self._pages is None:
            raise ValueError("BatchDecoder.fork: needs the paged layout (BatchDecoder(..., pages=P))")
        src, dst = self._slot(src), self._slot(dst)
        if self._pos[src] < 0 or self._pos[dst] >= 0 or src == dst:
            raise ValueError(f"BatchDecoder.fork: src must be active and dst idle (positions {self._pos[src]} and {self._pos[dst]})")
        p = self._pos[src]
        copy = self._pages.fork(src, dst, p)
        with torch.no_grad():
            if copy is not None:
                self._k[:, copy[1]].copy_(self._k[:, copy[0]])
                self._v[:, copy[1]].copy_(self._v[:, copy[0]])
            self.block_table[dst].copy_(torch.tensor(self._pages.tables[dst], dtype=torch.int32))
        self._set_pos(dst, p)

    @property
    def positions(self):
        """The position each slot's next step writes, -1 for an idle slot (host copy of the device positions)."""
        return list(self._pos)

    def prefill(self, slot, input_ids):
        """Run the prompt [1, T] (or [T]) alone through the model's own forward, copy its KV cache into `slot` and set the slot's
        position to T; returns the logits of the last position."""
        return self._prefill("BatchDecoder.prefill", self._slot(slot), input_ids)

    def extend(self, slot, input_ids):
        """Append the tokens input_ids (1-D) to `slot` at its position (0 for an idle slot) on the decoder's own kernels, as
        SequenceDecoder.extend does, advance the slot's position by T and return the logits of the last token.  It reads and writes
        nothing of the other slots, so it may run between steps while they keep their state.  Raises ValueError, with nothing written,
        for a bad slot, an empty or non-1-D prompt or one that does not fit in max_len."""
        return self._extend("BatchDecoder.extend", [(self._slot(slot), input_ids)])[0]

    def extend_many(self, slots, prompts):
        """Append prompts[i] (1-D token ids) to slots[i] at its position (0 for an idle slot) for every i in one run through the model,
        advance each slot's position by its prompt's length and return the logits of each prompt's last token, [len(slots), vocab] in
        the given order.  This is extend() for several slots at once: the prompts' tokens go through the projections together,
        EXTEND_CHUNK rows per pass (a prompt may span passes), and each layer's attention runs every prompt's rows of the pass in one
        quant_cuda.attn_extend_batch call (a pass with one prompt's rows runs attn_extend, as extend() does).  A slot's cache ends up
        bitwise as extend() would leave it, and its logits are those of its own prompt (the projections of a row do not depend on the
        other rows' values, though the kernel that runs them depends on how many rows a pass holds).  Slots not named are neither
        read nor written, so the others keep their state; forked slots may take different turns.  Admitting several short prompts
        this way reads the weights once per pass instead of once per prompt.
        Raises ValueError, with nothing written, unless slots and prompts have one length in 1..batch, the slots are distinct valid
        slots, and every prompt is a non-empty 1-D integer tensor that fits in max_len at its slot's position (the message names the
        prompt's index); paged, RuntimeError naming the slots, with nothing changed, when the pool cannot hold every prompt's pages."""
        slots, prompts = list(slots), list(prompts)
        if len(slots) != len(prompts) or not 1 <= len(slots) <= self.batch:
            raise ValueError(f"BatchDecoder.extend_many: {len(slots)} slots and {len(prompts)} prompts; want one length in 1..{self.batch}")
        slots = [self._slot(s) for s in slots]
        if len(set(slots)) != len(slots):
            raise ValueError(f"BatchDecoder.extend_many: the slots must be distinct (got {slots})")
        return self._extend("BatchDecoder.extend_many", list(zip(slots, prompts)), named=True)

    def step(self, token_ids):
        """Feed token_ids ([batch] ints or a device tensor; only the active slots' entries matter) at each active slot's position;
        returns the next-token logits [batch, vocab], a static buffer that the next step overwrites."""
        t = torch.as_tensor(token_ids)
        if t.numel() != self.batch:
            raise ValueError(f"BatchDecoder.step: {t.numel()} token ids for {self.batch} slots")
        self.tok.copy_(t.reshape(self.batch))
        self._replay()
        return self.logits

    def generate(self, prompts, max_new_tokens, eos_token_id=None, *, temperature=0.0, top_k=0, top_p=1.0, seed=0):
        """Each of the 1..batch prompts (1-D token ids, or [1, T]) followed by up to max_new_tokens tokens, ending after its first EOS
        (eos_token_id: an int or a list) if one comes; prompt i runs in slot i, the other slots stay idle.  Every prompt and
        max_new_tokens - 1 steps must fit in max_len.  Returns one 1-D tensor per prompt (prompt + new tokens), in order.
        Greedy by default; temperature > 0 samples as SequenceDecoder.generate does.  Each keyword is a scalar or a list of one value
        per prompt (temperature 0 keeps that prompt greedy); a scalar seed s gives prompt i the seed s + i.  A prompt's tokens depend on
        its own prompt, parameters and seed only.  Bad values raise ValueError before anything runs (see _sampling)."""
        prompts = [torch.as_tensor(p).reshape(-1) for p in prompts]
        if not 1 <= len(prompts) <= self.batch:
            raise ValueError(f"BatchDecoder.generate: {len(prompts)} prompts, the decoder takes 1 to {self.batch}")
        sampling = _sampling("BatchDecoder.generate", len(prompts), temperature, top_k, top_p, seed)
        if not isinstance(max_new_tokens, int) or max_new_tokens < 1:
            raise ValueError(f"BatchDecoder.generate: max_new_tokens must be a positive int (got {max_new_tokens!r})")
        for i, p in enumerate(prompts):
            if p.numel() < 1:
                raise ValueError(f"BatchDecoder.generate: prompt {i} is empty")
            if p.numel() + max_new_tokens - 1 > self.max_len:
                raise ValueError(f"BatchDecoder.generate: prompt {i} has {p.numel()} tokens and {max_new_tokens} new ones need "
                                 f"{p.numel() + max_new_tokens - 1} cache positions, max_len is {self.max_len}")
        eos = _eos_set(eos_token_id)
        self.reset()
        out, length = self._generate("BatchDecoder.prefill", prompts, max_new_tokens, eos, sampling)
        return [torch.cat([p.to(self.device), out[i, :length[i]]]) for i, p in enumerate(prompts)]
