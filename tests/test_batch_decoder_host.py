"""CPU tests of runtime.BatchDecoder's host side: every rejection that needs no device (ValueError naming the reason, before anything is
allocated or stacked) on models built on the CPU from HF configs, and the argument checks of generate()."""
import pytest
import torch

pytest.importorskip("transformers")

from test_decoder_host import REJECT, quantized  # noqa: E402

from squeezellm_b200.quant import QuantLinearLUT  # noqa: E402
from squeezellm_b200.runtime import BatchDecoder  # noqa: E402


def _unstacked(model):
    return all(m._sibling_group is None for m in model.modules() if isinstance(m, QuantLinearLUT))


@pytest.mark.parametrize("dtype,batch,frag", [
    (torch.float16, 1, r"batch must be an int in 2\.\.63 for a torch.float16 model \(got 1\); decode one sequence with SequenceDecoder"),
    (torch.float16, 0, r"batch must be an int in 2\.\.63 for a torch.float16 model \(got 0\)$"),
    (torch.float16, 64, r"batch must be an int in 2\.\.63 for a torch.float16 model \(got 64\)$"),
    (torch.bfloat16, 1, r"batch must be an int in 2\.\.79 for a torch.bfloat16 model \(got 1\); decode one sequence with SequenceDecoder"),
    (torch.bfloat16, 80, r"batch must be an int in 2\.\.79 for a torch.bfloat16 model \(got 80\)$"),
    (torch.float16, 2.0, r"batch must be an int in 2\.\.63 for a torch.float16 model \(got 2\.0\)$"),
])
def test_rejects_a_batch_out_of_range(dtype, batch, frag):
    model = quantized(dtype=dtype)
    with pytest.raises(ValueError, match="BatchDecoder: " + frag):
        BatchDecoder(model, 32, batch)
    assert _unstacked(model)


@pytest.mark.parametrize("dtype,batch", [(torch.float16, 2), (torch.float16, 63), (torch.bfloat16, 64), (torch.bfloat16, 79)])
def test_accepts_the_batch_range_then_wants_a_gpu(dtype, batch):
    model = quantized(dtype=dtype)
    with pytest.raises(ValueError, match=r"BatchDecoder: the model must be on one GPU \(its tensors are on \['cpu'\]\)"):
        BatchDecoder(model, 32, batch)
    assert _unstacked(model)


@pytest.mark.parametrize("make,frag", REJECT, ids=["class", "fp32", "dense_layer", "mixed_bits", "trained", "mistral_window",
                                                   "qwen2_window", "head_dim_32", "head_dim_256", "act"])
def test_rejections_of_the_shared_layout(make, frag):
    model = make()
    with pytest.raises(ValueError, match="BatchDecoder: .*" + frag):
        BatchDecoder(model, 32, 4)


@pytest.mark.parametrize("max_len", [0, -3, 2.5])
def test_rejects_a_bad_max_len(max_len):
    with pytest.raises(ValueError, match="BatchDecoder: max_len must be a positive int"):
        BatchDecoder(quantized(), max_len, 4)


def test_rejects_a_quantized_lm_head_the_rows_kernel_does_not_take():
    model = quantized(quant_head=True, vocab_size=130)  # out_features not a multiple of 4
    with pytest.raises(ValueError, match=r"BatchDecoder: lm_head \(256 -> 130\) does not fit the multi-row LUT-GEMV"):
        BatchDecoder(model, 32, 4)
    assert _unstacked(model)


def test_rejects_a_layer_too_wide_for_the_rows_kernel():
    from squeezellm_b200.quant import FUSED_LIMITS
    wide = FUSED_LIMITS["rows_max_in_features"] + 32
    model = quantized(num_hidden_layers=1, intermediate_size=wide)
    with pytest.raises(ValueError, match=rf"BatchDecoder: layers\.0\.mlp\.down_proj \({wide} -> 256\) does not fit the multi-row "
                                         rf"LUT-GEMV \(out_features a multiple of 4, in_features up to {wide - 32}\)"):
        BatchDecoder(model, 32, 4)
    assert _unstacked(model)


# ---- generate()'s argument checks, made before anything runs ----
def _decoder(batch=4, max_len=32):
    dec = BatchDecoder.__new__(BatchDecoder)  # the checks read only batch and max_len
    dec.batch, dec.max_len = batch, max_len
    return dec


@pytest.mark.parametrize("prompts,n,frag", [
    ([], 4, r"0 prompts, the decoder takes 1 to 4"),
    ([[1, 2]] * 5, 4, r"5 prompts, the decoder takes 1 to 4"),
    ([[1, 2]], 0, r"max_new_tokens must be a positive int \(got 0\)"),
    ([[1, 2]], 2.0, r"max_new_tokens must be a positive int \(got 2\.0\)"),
    ([[1, 2], []], 4, r"prompt 1 is empty"),
    ([[1], list(range(30))], 4, r"prompt 1 has 30 tokens and 4 new ones need 33 cache positions, max_len is 32"),
])
def test_generate_rejects(prompts, n, frag):
    with pytest.raises(ValueError, match="BatchDecoder.generate: " + frag):
        _decoder().generate(prompts, n)


@pytest.mark.parametrize("slot", [-1, 4, 1.0])
def test_slots_are_checked(slot):
    with pytest.raises(ValueError, match=r"slot must be an int in 0\.\.3"):
        _decoder().release(slot)
    with pytest.raises(ValueError, match=r"slot must be an int in 0\.\.3"):
        _decoder().prefill(slot, [1, 2])
