"""CPU tests of speculative decoding's host side in runtime: the prompt-lookup drafter (PromptLookup) on hand-made histories, the accept
rule (accept_length), and every rejection of SequenceDecoder(speculate=), verify(), rewind() and generate(draft=) that needs no device
(ValueError naming the reason, before anything is allocated, stacked or written)."""
import pytest
import torch

pytest.importorskip("transformers")

from test_decoder_host import quantized  # noqa: E402

from squeezellm_b200.quant import QuantLinearLUT  # noqa: E402
from squeezellm_b200.runtime import PromptLookup, SequenceDecoder, accept_length  # noqa: E402


# ---- the prompt-lookup drafter ----
def test_lookup_prefers_the_longest_ngram():
    # suffix (7, 1, 2): its 3-gram occurred at 4..6 (followed by 9, 9); its 2-gram (1, 2) occurred later at 8..9 (followed by 5)
    d = PromptLookup([3, 3, 3, 3, 7, 1, 2, 9, 1, 2, 5, 0, 7, 1, 2], k=2)
    assert d.propose() == [9, 1]


def test_lookup_falls_back_to_two_tokens_and_takes_the_most_recent():
    d = PromptLookup([1, 2, 3, 8, 1, 2, 4, 6, 1, 2], k=3)  # no earlier (8, 1, 2) ... (6, 1, 2); (1, 2) last at 4..5
    assert d.propose() == [4, 6, 1]


def test_lookup_finds_nothing():
    assert PromptLookup([1, 2, 3, 4, 5], k=4).propose() == []
    assert PromptLookup([], k=4).propose() == []
    assert PromptLookup([7, 7], k=4).propose() == []  # the suffix (7, 7) is the whole history: no earlier occurrence


def test_lookup_gives_fewer_than_k_near_the_end():
    d = PromptLookup([5, 6, 7, 5, 6], k=4)  # (5, 6) at 0..1, followed by 7, 5, 6 only
    assert d.propose() == [7, 5, 6]
    d = PromptLookup([1, 1, 1], k=4)  # (1, 1) at 0..1 followed by one 1
    assert d.propose() == [1]


def test_lookup_extends_incrementally_as_a_rescan_would():
    import random
    rng = random.Random(3)
    toks = [rng.randrange(6) for _ in range(300)]
    d = PromptLookup(toks[:10], k=5)
    i = 10
    while i < len(toks):
        j = min(len(toks), i + rng.randrange(1, 5))
        d.extend(toks[i:j])
        i = j
        fresh = PromptLookup(toks[:i], k=5)
        assert d.propose() == fresh.propose()
        want = []  # the definition, by a scan: n = 3 then 2, the most recent earlier occurrence of the suffix
        for n in (3, 2):
            hits = [s for s in range(i - n) if toks[s:s + n] == toks[i - n:i]]
            if hits:
                want = toks[hits[-1] + n:min(i, hits[-1] + n + 5)]
                break
        assert d.propose() == want


# ---- the accept rule ----
@pytest.mark.parametrize("drafts,draws,n", [
    ([], [4], 0),
    ([4, 5, 6], [4, 5, 6, 7], 3),
    ([4, 5, 6], [4, 9, 6, 7], 1),
    ([4, 5, 6], [0, 5, 6, 7], 0),
    ([4, 5], [4, 5, 1, 1], 2),   # fewer drafts than rows: the padding rows are never looked at
])
def test_accept_length(drafts, draws, n):
    assert accept_length(drafts, draws) == n


# ---- rejections ----
def _unstacked(model):
    return all(m._sibling_group is None for m in model.modules() if isinstance(m, QuantLinearLUT))


@pytest.mark.parametrize("k", [-1, 16, 2.0, True, "3"])
def test_rejects_a_bad_speculate(k):
    model = quantized()
    with pytest.raises(ValueError, match=r"SequenceDecoder: speculate must be an int in 0\.\.15 \(got "):
        SequenceDecoder(model, 32, speculate=k)
    assert _unstacked(model)


def test_rejects_a_quantized_lm_head_the_rows_kernel_does_not_take():
    model = quantized(quant_head=True, vocab_size=130)  # out_features not a multiple of 4
    with pytest.raises(ValueError, match=r"SequenceDecoder: lm_head \(256 -> 130\) does not fit the multi-row LUT-GEMV"):
        SequenceDecoder(model, 32, speculate=3)
    assert _unstacked(model)
    with pytest.raises(ValueError, match="the model must be on one GPU"):  # without speculation the one-GEMV kernels take it
        SequenceDecoder(model, 32)


def test_rejects_a_layer_too_wide_for_the_rows_kernel():
    from squeezellm_b200.quant import FUSED_LIMITS
    wide = FUSED_LIMITS["rows_max_in_features"] + 32
    model = quantized(num_hidden_layers=1, intermediate_size=wide)
    with pytest.raises(ValueError, match=rf"SequenceDecoder: layers\.0\.mlp\.down_proj \({wide} -> 256\) does not fit the multi-row "
                                         rf"LUT-GEMV \(out_features a multiple of 4, in_features up to {wide - 32}\)"):
        SequenceDecoder(model, 32, speculate=1)
    assert _unstacked(model)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_accepts_speculate_then_wants_a_gpu(dtype):
    model = quantized(dtype=dtype)
    with pytest.raises(ValueError, match=r"SequenceDecoder: the model must be on one GPU"):
        SequenceDecoder(model, 32, speculate=15)
    assert _unstacked(model)


def _decoder(speculate=3, max_len=32, position=10):
    dec = SequenceDecoder.__new__(SequenceDecoder)  # the checks read only these
    dec.speculate, dec.max_len, dec._pos = speculate, max_len, [position]
    return dec


@pytest.mark.parametrize("ids,frag", [
    ([1, 2, 3], r"3 token ids, the verify step takes speculate \+ 1 = 4"),
    ([1, 2, 3, 4, 5], r"5 token ids, the verify step takes speculate \+ 1 = 4"),
    ([1.0, 2.0, 3.0, 4.0], r"token_ids must hold integer token ids \(got torch.float32\)"),
])
def test_verify_rejects(ids, frag):
    with pytest.raises(ValueError, match="SequenceDecoder.verify: " + frag):
        _decoder().verify(ids)


def test_verify_rejects_what_does_not_fit_and_a_decoder_without_speculation():
    with pytest.raises(ValueError, match=r"SequenceDecoder.verify: 4 tokens at position 29 need 33 cache positions, max_len is 32"):
        _decoder(position=29).verify([1, 2, 3, 4])
    with pytest.raises(ValueError, match=r"SequenceDecoder.verify: the decoder was built with speculate=0"):
        _decoder(speculate=0).verify([1])


@pytest.mark.parametrize("n", [-1, 11, 3.0, True])
def test_rewind_rejects(n):
    with pytest.raises(ValueError, match=r"SequenceDecoder.rewind: position must be an int in 0\.\.10"):
        _decoder().rewind(n)


def test_generate_rejects_a_draft_without_speculation_or_not_callable():
    with pytest.raises(ValueError, match=r"SequenceDecoder.generate: draft needs a decoder built with speculate > 0"):
        _decoder(speculate=0).generate([1, 2], 4, draft=lambda toks: [])
    with pytest.raises(ValueError, match=r"SequenceDecoder.generate: draft must be a callable"):
        _decoder().generate([1, 2], 4, draft=[1, 2])


@pytest.mark.parametrize("out,frag", [
    ([1, 128], r"draft returned 128, not a token id in \[0, 128\)"),
    ([-1], r"draft returned -1, not a token id in \[0, 128\)"),
    ([1, 2.0], r"draft returned 2\.0, not a token id"),
    ([True], r"draft returned True, not a token id"),
    (None, r"draft must return a list of token ids \(got NoneType\)"),
    (5, r"draft must return a list of token ids \(got int\)"),
])
def test_a_bad_drafter_output_is_rejected(out, frag):
    with pytest.raises(ValueError, match="SequenceDecoder.generate: " + frag):
        SequenceDecoder._check_draft(out, 128)


def test_a_drafter_output_is_taken_as_ints():
    import numpy as np
    assert SequenceDecoder._check_draft((np.int64(3), 4), 128) == [3, 4]
    assert SequenceDecoder._check_draft(torch.tensor([5, 6]), 128) == [5, 6]
    assert SequenceDecoder._check_draft([], 128) == []
