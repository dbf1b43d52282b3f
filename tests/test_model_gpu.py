"""Every QuantLinearLUT call of real transformers models on the GPU against the fp64 oracle, per element: the code above the kernels
(QuantLinearLUT.forward's dispatch, sibling stacking, the autograd functions, codebook training) with the inputs a model gives it -
3-D activations, [B, 1, h] decode batches, GQA sibling slices (q / k / v of widths 1024 / 256 / 256), bf16 and fp32 models, and fp32
outputs after a bias that send the next layers down the fp32 routes.

Models (random init from a config, eager attention, nothing downloaded), built in the target dtype, then loaded from a reference-
format checkpoint (checkpoint.load_quantized: oracle.make_layer layers, CSR 0.45 %, 10 non-zero dense rows), then .cuda(), usually
then fusion.fuse_siblings.  The codebooks, outliers and dense rows are scaled to entries of about 1 / sqrt(in_features), so that
activations stay O(1) through the blocks:
  * A: Llama, hidden 1024, intermediate 2816, 2 layers, 8 heads, 2 KV heads, vocab 512; at 4 and at 3 bits.
  * B: one 7B-shaped Llama decoder layer (hidden 4096, intermediate 11008, 32 heads), vocab 256, 4 bits.
  * C: Qwen2 (bias on q / k / v, none on o), otherwise A, 4 bits.  Its lm_head is quantized too: a biased batch call returns fp32
    (out.to(dtype) + fp32 bias, as the reference's quant.py), every later layer of an fp16 model then gets fp32 x, and HF's fp16
    nn.Linear lm_head would reject the fp32 hidden state.

Per call: a forward hook on every QuantLinearLUT records (x, y) as HF passed and received them; y is checked against
x64 @ W (+ b) with util.bound_ratio, W the dense fp64 weight of the oracle (backward_ref.dense_w_f64; never the dequantize kernel),
the bias inside the rounded sum for 1-row calls and added after the rounding otherwise.  The x the layer actually received is
used, so no error carries over from earlier layers.  A spy on the quant_cuda bindings records the routes each case reaches and
the case asserts the set it claims to cover.  End to end, beside it: the logits of the model against an fp64 twin (the same HF
class in float64 holding W.T), next to the logits of a dense model in the same dtype (the twin's weights rounded, cuBLAS).

Backward: input gradients through the model (fused and unfused, fp16 and bf16, both lutgemm_t paths) per element against
dy . W^T; codebook training: every lut_grad call against lut_grad_ref, then one Adam step followed at once by a decode step."""
import copy

import numpy as np
import pytest
import torch

from backward_ref import dense_w_f64
from lut_grad_ref import lut_grad_f64
from test_lut_grad_gpu import check as check_lut_grad
from util import OUT_ROUNDING, abs_layer, bound_ratio, orc

pytestmark = pytest.mark.gpu

transformers = pytest.importorskip("transformers")

DTYPES = {"fp16": torch.float16, "bf16": torch.bfloat16, "fp32": torch.float32}
SPEC = {  # kind: (config class, config kwargs, bits, lm_head quantized)
    "A4": ("LlamaConfig", dict(hidden_size=1024, intermediate_size=2816, num_hidden_layers=2, num_attention_heads=8,
                               num_key_value_heads=2, vocab_size=512), 4, False),
    "A3": ("LlamaConfig", dict(hidden_size=1024, intermediate_size=2816, num_hidden_layers=2, num_attention_heads=8,
                               num_key_value_heads=2, vocab_size=512), 3, False),
    "B": ("LlamaConfig", dict(hidden_size=4096, intermediate_size=11008, num_hidden_layers=1, num_attention_heads=32,
                              num_key_value_heads=32, vocab_size=256), 4, False),
    "C": ("Qwen2Config", dict(hidden_size=1024, intermediate_size=2816, num_hidden_layers=2, num_attention_heads=8,
                              num_key_value_heads=2, vocab_size=512), 4, True),
}


def _config(kind):
    cls, kw, _, _ = SPEC[kind]
    return getattr(transformers, cls)(max_position_embeddings=256, attn_implementation="eager", **kw)


def _model_class(kind):
    return transformers.Qwen2ForCausalLM if SPEC[kind][0] == "Qwen2Config" else transformers.LlamaForCausalLM


class Bank:
    """The numpy layer dicts of one model kind (oracle.make_layer, scaled) and their dense fp64 weights W [K, N] and |W| on the GPU,
    made once per test module."""

    def __init__(self, kind):
        from squeezellm_b200 import checkpoint as ck
        _, _, bits, quant_head = SPEC[kind]
        torch.manual_seed(0)
        model = _model_class(kind)(_config(kind))
        self.kind, self.bits = kind, bits
        self.L, self.W, self.Wa = {}, {}, {}
        for i, (name, lin) in enumerate(sorted(ck.find_linear_layers(model).items())):
            if name == "lm_head" and not quant_head:
                continue
            K, N = lin.in_features, lin.out_features
            L = orc.make_layer(bits, K, N, sparsity=0.0045, topX=10, seed=1000 + 17 * i, nonzero_full_rows=True,
                               bias=lin.bias is not None)
            s = 1.0 / np.sqrt(K)  # entries of about 1 / sqrt(K): |y| ~ |x|
            L["lookup_table"] = (L["lookup_table"] * (s / 0.02)).astype(np.float32)
            L["vals"] = (L["vals"] * (s / 0.1)).astype(np.float32)
            L["full_rows"] = (L["full_rows"] * (s / 0.05)).astype(np.float32)
            self.L[name] = L
            self.W[name] = torch.from_numpy(dense_w_f64(L)).cuda()
            self.Wa[name] = torch.from_numpy(dense_w_f64(abs_layer(L))).cuda()
        del model
        self._w16 = {}

    def w_fp16_lut(self, name):
        """W and |W| with the codebook rounded to fp16 (the one-GEMV kernel's fp16 table mode)."""
        if name not in self._w16:
            L = dict(self.L[name], lookup_table=self.L[name]["lookup_table"].astype(np.float16).astype(np.float32))
            self._w16[name] = (torch.from_numpy(dense_w_f64(L)).cuda(), torch.from_numpy(dense_w_f64(abs_layer(L))).cuda())
        return self._w16[name]


_banks = {}


@pytest.fixture(scope="module")
def banks():
    yield _banks
    _banks.clear()
    torch.cuda.empty_cache()


def bank(banks, kind):
    if kind not in banks:
        banks[kind] = Bank(kind)
    return banks[kind]


def build(bk, dtype, fuse=True):
    """The quantized model of `bk` in `dtype`: built in dtype, loaded from the reference-format checkpoint, moved to the GPU, siblings
    stacked when `fuse`.  -> (model, {module: layer name}, sibling groups)."""
    from squeezellm_b200 import checkpoint as ck, fusion
    from squeezellm_b200.quant import QuantLinearLUT
    torch.manual_seed(0)
    model = _model_class(bk.kind)(_config(bk.kind)).to(dtype).eval()
    state = {k: v.clone() for k, v in model.state_dict().items()}
    for name, L in bk.L.items():
        del state[name + ".weight"]
        for k in ("qweight", "lookup_table", "rows", "cols", "vals", "full_rows", "full_row_indices", "bias"):
            if L.get(k) is not None:
                state[f"{name}.{k}"] = torch.from_numpy(L[k])
        state["sparse_threshold." + name] = len(L["vals"])
    res = ck.load_quantized(model, state, bk.bits, include_sparse=True, topX=10, skip=() if SPEC[bk.kind][3] else ("lm_head",))
    assert not res.missing_keys and not res.unexpected_keys, res
    model = model.cuda()
    names = {m: n for n, m in model.named_modules() if isinstance(m, QuantLinearLUT)}
    assert set(names.values()) == set(bk.L)
    groups = fusion.fuse_siblings(model) if fuse else []
    return model, names, groups


def twin_of(bk, model):
    """The fp64 twin: the same HF class in float64 with nn.Linear weights W.T and the same biases, embeddings, norms and lm_head."""
    twin = _model_class(bk.kind)(_config(bk.kind)).to(torch.float64).eval()
    src = model.state_dict()
    sd = {}
    for k in twin.state_dict():
        layer, leaf = k.rsplit(".", 1)
        if layer in bk.L:
            sd[k] = bk.W[layer].t().contiguous() if leaf == "weight" else torch.from_numpy(bk.L[layer]["bias"]).double()
        else:
            sd[k] = src[k].double()
    twin.load_state_dict(sd)
    return twin.cuda()


# ---- the spy on the extension ------------------------------------------------------------------------------------------------
def route_name(binding):
    if binding.startswith("vecquant"):
        return "_batched" if binding.endswith("_batched") else "symbols"
    return binding


@pytest.fixture
def spy(monkeypatch):
    """Names of the quant_cuda bindings called, in order."""
    from squeezellm_b200 import quant
    calls = []
    for n in dir(quant.quant_cuda):
        if n.startswith(("lutgemv", "lutgemm", "vecquant", "lut_grad")):
            real = getattr(quant.quant_cuda, n)
            monkeypatch.setattr(quant.quant_cuda, n, (lambda real, n: lambda *a, **kw: (calls.append((n, kw.get("path"))),
                                                                                          real(*a, **kw))[1])(real, n))
    return calls


@pytest.fixture
def record(request):
    return lambda name, value: request.node.user_properties.append((name, value))


@pytest.fixture
def modes():
    """Restores the process-wide switches the cases change."""
    from squeezellm_b200.quant import QuantLinearLUT, quant_cuda
    yield QuantLinearLUT, quant_cuda
    QuantLinearLUT.use_fused = True
    quant_cuda.set_lut_mode("exact")


# ---- the per-call truth ------------------------------------------------------------------------------------------------------
class Recorder:
    """Forward hooks on every QuantLinearLUT of a model: (layer name, launched width, x, y) of every call."""

    def __init__(self, model, names):
        self.calls = []
        self.handles = []
        for m, n in names.items():
            self.handles.append(m.register_forward_hook(lambda mod, inp, out, n=n: self.calls.append((n, self._width(mod), inp[0], out))))

    @staticmethod
    def _width(mod):
        g = mod._sibling_group
        return g[0].layer.outfeatures if g is not None else mod.outfeatures

    def remove(self):
        for h in self.handles:
            h.remove()


def check_call(bk, name, width, x, y, lut_fp16=False, L=None):
    """bound_ratio of one recorded call.  L: the layer dict to take the truth from (default: bk.L[name])."""
    L = bk.L[name] if L is None else L
    K, N = L["infeatures"], L["outfeatures"]
    M = x.numel() // K
    x = x.detach()
    b = L.get("bias")
    assert y.shape == x.shape[:-1] + (N,), (name, y.shape, x.shape)
    want_dtype = x.dtype if M == 1 or b is None else torch.result_type(x, torch.zeros(1))
    assert y.dtype == want_dtype, (name, M, x.dtype, y.dtype)
    if L is not bk.L[name]:
        W, Wa = torch.from_numpy(dense_w_f64(L)).cuda(), torch.from_numpy(dense_w_f64(abs_layer(L))).cuda()
    elif lut_fp16 and M == 1 and x.dtype == torch.float16 and width >= 64:
        W, Wa = bk.w_fp16_lut(name)  # lutgemv.cu (lutgemv_fused): the fp16 table serves fp16 x on layers of at least one 64-column strip
    else:
        W, Wa = bk.W[name], bk.Wa[name]
    x64 = x.reshape(M, K).double()
    want = x64 @ W
    S = x64.abs() @ Wa
    rounded = want
    if b is not None:
        b64 = torch.from_numpy(b).double().cuda()
        want, S = want + b64, S + b64.abs()
        rounded = want if M == 1 else rounded
    r, eta = OUT_ROUNDING[str(x.dtype).split(".")[1]]
    return bound_ratio(y.detach().reshape(M, N).double().cpu().numpy(), want.cpu().numpy(), S.cpu().numpy(), rounded.cpu().numpy(),
                       r, eta=eta)


def check_calls(bk, rec, lut_fp16=False):
    worst = 0.0
    for name, width, x, y in rec.calls:
        ratio = check_call(bk, name, width, x, y, lut_fp16)
        assert ratio <= 1.0, (name, tuple(x.shape), x.dtype, ratio)
        worst = max(worst, ratio)
    n = len(rec.calls)
    rec.calls.clear()
    return worst, n


# ---- forward cases -------------------------------------------------------------------------------------------------------------
# (model, dtype, variant, prefill rows, decode batches, routes that must be hit)
CASES = [
    ("A4", "fp16", "", [17, 64], [1, 5, 63, 64], {"lutgemv_rows", "lutgemm_fused", "lutgemv_fused"}),
    ("A4", "bf16", "", [17, 80], [1, 79, 80], {"lutgemv_rows_bf16", "lutgemm_fused", "lutgemv_fused"}),
    ("A4", "fp32", "", [17, 128], [1], {"_batched", "lutgemm_fused_f32", "lutgemv_fused"}),
    ("A4", "fp16", "unfused", [17], [1, 5], {"symbols", "_batched"}),
    ("A4", "fp16", "lut16", [64], [1, 5], {"lutgemm_fused", "lutgemv_fused", "lutgemv_rows"}),
    ("A3", "fp16", "", [17, 64], [1, 5, 63, 64], {"lutgemv_rows", "lutgemm_fused", "lutgemv_fused"}),
    ("A3", "bf16", "", [17, 80], [1, 79, 80], {"lutgemv_rows_bf16", "lutgemm_fused", "lutgemv_fused"}),
    ("B", "fp16", "", [17, 64], [1, 5, 63, 64], {"lutgemv_rows", "lutgemm_fused", "lutgemv_fused"}),
    ("B", "bf16", "", [17, 80], [1, 79, 80], {"lutgemv_rows_bf16", "lutgemm_fused", "lutgemv_fused"}),
    # C in fp16: q / k / v return fp32 for every batch (their bias), so o_proj, the MLP and the lm_head of that block and all later
    # layers see fp32 x and take the fp32 routes (fewer than 128 rows: the _batched symbols).  Prefill only: a 1-row decode step
    # returns fp16 q / k / v, and HF's attention rejects fp16 queries against the fp32 keys the prefill cached.
    ("C", "fp16", "", [17, 64], [], {"lutgemv_rows", "lutgemm_fused", "_batched"}),
    ("C", "fp32", "", [17, 128], [1], {"_batched", "lutgemm_fused_f32", "lutgemv_fused"}),
]
DECODE_PROMPT = 2  # tokens per sequence before the decode steps
DECODE_STEPS = 2


def _run(model, steps):
    """steps: [(input ids, reuse the cache)] -> list of fp64 logits, one per step."""
    out, cache = [], None
    for ids, cont in steps:
        o = model(input_ids=ids, past_key_values=cache if cont else None, use_cache=True)
        cache = o.past_key_values
        out.append(o.logits.double())
    return out


@pytest.mark.parametrize("kind,dtype,variant,prefill,decode,routes", CASES,
                         ids=[f"{k}-{d}{'-' + v if v else ''}" for k, d, v, *_ in CASES])
def test_every_call_of_a_model_against_the_oracle(banks, spy, modes, record, kind, dtype, variant, prefill, decode, routes):
    QuantLinearLUT, quant_cuda = modes
    bk = bank(banks, kind)
    dt = DTYPES[dtype]
    model, names, groups = build(bk, dt, fuse=variant != "unfused")
    vocab = model.config.vocab_size
    gen = torch.Generator().manual_seed(7)
    rec = Recorder(model, names)
    worst, ncalls, steps = 0.0, 0, []
    try:
        QuantLinearLUT.use_fused = variant != "unfused"
        if variant == "lut16":
            quant_cuda.set_lut_mode("fp16")
        with torch.no_grad():
            runs = [(torch.randint(0, vocab, (1, T), generator=gen), 0) for T in prefill] + \
                   [(torch.randint(0, vocab, (B, DECODE_PROMPT), generator=gen), DECODE_STEPS) for B in decode]
            for ids, n_dec in runs:
                ids = ids.cuda()
                launches = [g.launches for g in groups]
                o = model(input_ids=ids, use_cache=True)
                seq = [(ids, False)]
                for _ in range(n_dec):
                    nxt = o.logits[:, -1:].argmax(-1)
                    o = model(input_ids=nxt, past_key_values=o.past_key_values, use_cache=True)
                    seq.append((nxt, True))
                steps.append(seq)
                # one stacked launch per sibling set and step
                assert [g.launches - l for g, l in zip(groups, launches)] == [1 + n_dec] * len(groups)
                w, n = check_calls(bk, rec, lut_fp16=variant == "lut16")
                worst, ncalls = max(worst, w), ncalls + n
    finally:
        rec.remove()
        QuantLinearLUT.use_fused = True
        quant_cuda.set_lut_mode("exact")
    hit = {route_name(n) for n, _ in spy}
    record("routes", sorted(hit))
    record("bound_ratio", worst)
    record("calls_checked", ncalls)
    if variant == "unfused":
        assert hit == routes, hit  # the reference's 12 symbols only
    else:
        assert routes <= hit, (routes, hit)
    # end to end: the quantized model and a dense model in the same dtype against the fp64 twin, on the same tokens
    twin = twin_of(bk, model)
    dense = copy.deepcopy(twin).to(dt)
    err_q = err_d = 0.0
    with torch.no_grad():
        QuantLinearLUT.use_fused = variant != "unfused"
        if variant == "lut16":
            quant_cuda.set_lut_mode("fp16")
        try:
            for seq in steps:
                for lq, lt, ld in zip(_run(model, seq), _run(twin, seq), _run(dense, seq)):
                    err_q = max(err_q, (lq - lt).abs().max().item())
                    err_d = max(err_d, (ld - lt).abs().max().item())
        finally:
            QuantLinearLUT.use_fused = True
            quant_cuda.set_lut_mode("exact")
    record("err_quant", err_q)
    record("err_dense", err_d)
    assert err_q <= 2 * err_d, (err_q, err_d)


# ---- backward ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fuse", [False, True], ids=["unfused", "fused"])
@pytest.mark.parametrize("dtype", ["fp16", "bf16"])
def test_input_gradients_through_a_model(banks, spy, monkeypatch, record, dtype, fuse):
    """Cross-entropy through model A from inputs_embeds that require grad, at 17 and 96 rows (both sides of BWD_TC_MIN_ROWS):
    every dx = dy . W^T the layers compute, per element against the fp64 truth (the bound of test_backward_gpu.check).  A stacked
    layer's truth is its members' weights side by side.  dy is taken where _input_grad receives it, not from backward hooks on the
    members: those re-wrap x per module and would break the sibling cache's identity test."""
    from squeezellm_b200.quant import QuantLinearLUT
    bk = bank(banks, "A4")
    dt = DTYPES[dtype]
    model, names, groups = build(bk, dt, fuse=fuse)
    of_layer = {m: [n] for m, n in names.items()}
    for g in groups:
        of_layer[g.layer] = [names[m] for m in g.members]
    seen = []
    real = QuantLinearLUT._input_grad
    monkeypatch.setattr(QuantLinearLUT, "_input_grad", lambda self, dy: (lambda dx: (seen.append((self, dy, dx)), dx)[1])(real(self, dy)))
    worst = 0.0
    gen = torch.Generator().manual_seed(3)
    for T in (17, QuantLinearLUT.BWD_TC_MIN_ROWS):
        ids = torch.randint(0, model.config.vocab_size, (1, T + 1), generator=gen).cuda()
        emb = model.get_input_embeddings()(ids[:, :-1]).detach().requires_grad_()
        logits = model(inputs_embeds=emb).logits
        loss = torch.nn.functional.cross_entropy(logits.float().reshape(T, -1), ids[0, 1:])
        seen.clear()
        loss.backward()
        assert emb.grad is not None and torch.isfinite(emb.grad).all()
        assert len(seen) == (7 if not fuse else 4) * model.config.num_hidden_layers
        for layer, dy, dx in seen:
            W = torch.cat([bk.W[n] for n in of_layer[layer]], dim=1)
            Wa = torch.cat([bk.Wa[n] for n in of_layer[layer]], dim=1)
            dy64 = dy.reshape(-1, W.shape[1]).double()
            r, eta = OUT_ROUNDING[str(dx.dtype).split(".")[1]]
            assert dx.dtype == dy.dtype == dt
            ratio = bound_ratio(dx.double().cpu().numpy(), (dy64 @ W.t()).cpu().numpy(), (dy64.abs() @ Wa.t()).cpu().numpy(), r=r, eta=eta)
            assert ratio <= 1.0, (of_layer[layer], T, ratio)
            worst = max(worst, ratio)
        paths = {p for n, p in spy if n == "lutgemm_t"}
        assert paths == {"tc" if T >= QuantLinearLUT.BWD_TC_MIN_ROWS else "cuda"}, (T, paths)
        del spy[:]
    record("bound_ratio", worst)


# ---- codebook training -----------------------------------------------------------------------------------------------------------
def test_codebook_training_through_a_model_then_decode_after_adam(banks, spy, monkeypatch, record):
    """Unfused model A in fp16 with train_codebook(lookup_table, vals, full_rows) on every layer: every lut_grad call against
    lut_grad_ref per element (test_lut_grad_gpu.check).  Then one Adam step and, with no synchronisation in between, a 1-row decode
    step whose every call is checked against the oracle of the parameters' new values.

    The one-GEMV kernels read the codebook, the row pointers and the dense rows before griddepcontrol.wait, on the premise that
    nothing just before them in the stream writes weights.  This checks that stream order in the common pattern (optimizer step, then
    generate); one run cannot prove that no race exists."""
    from squeezellm_b200.quant import QuantLinearLUT
    bk = bank(banks, "A4")
    model, names, _ = build(bk, torch.float16, fuse=False)
    params = []
    for m in names:
        params += m.train_codebook(lookup_table=True, vals=True, full_rows=True)
    seen = []
    real = QuantLinearLUT._codebook_grad
    monkeypatch.setattr(QuantLinearLUT, "_codebook_grad",
                        lambda self, x, dy, want: (lambda g: (seen.append((self, x, dy, want, g)), g)[1])(real(self, x, dy, want)))
    ids = torch.randint(0, model.config.vocab_size, (1, 33), generator=torch.Generator().manual_seed(5)).cuda()
    logits = model(input_ids=ids[:, :-1]).logits
    loss = torch.nn.functional.cross_entropy(logits.float().reshape(32, -1), ids[0, 1:])
    loss.backward()
    assert len(seen) == len(names)
    for layer, x, dy, want, g in seen:
        L = bk.L[names[layer]]
        got = {k: v for k, v in zip(("lookup_table", "vals", "full_rows"), g) if k in want}
        assert set(got) == {"lookup_table", "vals", "full_rows"}
        check_lut_grad(got, lut_grad_f64(L, x.detach(), dy, device="cuda"), names[layer])
    assert {n for n, _ in spy} >= {"lut_grad", "lutgemm_t"}
    opt = torch.optim.Adam(params, lr=1e-3)
    rec = Recorder(model, names)
    try:
        opt.step()
        with torch.no_grad():  # immediately: no synchronisation between the step and the decode launches
            model(input_ids=ids[:, :1])
        torch.cuda.synchronize()
    finally:
        rec.remove()
    assert len(rec.calls) == len(names)
    worst = 0.0
    for name, width, x, y in rec.calls:
        m = next(mm for mm, n in names.items() if n == name)
        L = dict(bk.L[name], **{k: getattr(m, k).detach().cpu().numpy() for k in ("lookup_table", "vals", "full_rows")})
        assert not np.array_equal(L["lookup_table"], bk.L[name]["lookup_table"])
        ratio = check_call(bk, name, width, x, y, L=L)
        assert ratio <= 1.0, (name, ratio)
        worst = max(worst, ratio)
    record("bound_ratio", worst)
