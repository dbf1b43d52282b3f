"""Quantize a model on the GPU into QuantLinearLUT layers: the reference's offline pipeline (quantization/nuq.py,
squeezellm/outliers.py, quantization/generate_outlier_config.py, squeezellm/quant.py pack2) restated on top of the
`quant_cuda` extension.

  * `kmeans_codebook`: the per-output-channel weighted k-means of nuq.py:50-58,164-176, solved EXACTLY by a dynamic program
    on the sorted row (quant_cuda.kmeans1d; DESIGN.md section 3.13) instead of one seeded sklearn KMeans per row on the CPU.
    Its objective is never above sklearn's, and the result is deterministic.
  * `outlier_threshold`: the IQR rule of generate_outlier_config.py:47-53.
  * `split_outliers`: the sensitivity and threshold masks of outliers.py:14-23,52-60.
  * `quantize_linear` / `quantize_model`: the codebook fit, then the pack of quant.py:97-208 on the device (quant_cuda.pack_indices
    and a CSR of outlier minus zero centroid); buffers bit-identical to QuantLinearLUT.pack2 on the same inputs.
    `checkpoint.save_checkpoint` writes the result in the reference's format.
  * `dequantize_model`: the way back, every QuantLinearLUT replaced by an nn.Linear holding its dense weight
    (QuantLinearLUT.to_linear, quant_cuda.dequantize), e.g. to export a fine-tuned model as a plain dense checkpoint.
  * `fisher_information`: the first stage, the weights of the k-means: the diagonal of the empirical Fisher information, the sum
    over calibration sequences of each sequence's squared weight gradient (quant_cuda.fisher_accumulate, DESIGN.md section 3.15).
    Its result is the `fisher_state` quantize_model takes, so fisher_information -> quantize_model -> save_checkpoint turns a
    dense model into a SqueezeLLM checkpoint.
"""
import torch

from .checkpoint import find_linear_layers
from .quant import QuantLinearLUT, quant_cuda

__all__ = ["kmeans_codebook", "outlier_threshold", "split_outliers", "quantize_linear", "quantize_model", "dequantize_model",
           "fisher_information"]

_FISHER_DTYPES = (torch.float16, torch.bfloat16)  # the operand types of quant_cuda.fisher_accumulate


def kmeans_codebook(weight, sample_weight, bits):
    """Per-row exact weighted k-means with 2^bits clusters: weight, sample_weight [N, K] CUDA tensors ->
    (lookup_table fp32 [N, 2^bits] non-decreasing, labels uint8 [N, K] = nearest centroid, ties to the lower index).
    A row whose sample weights are all zero is weighted uniformly (nuq.py:174-175)."""
    if bits not in (3, 4):
        raise ValueError(f"kmeans_codebook: bits={bits} must be 3 or 4")
    if not (torch.is_tensor(weight) and torch.is_tensor(sample_weight)):
        raise ValueError("kmeans_codebook: weight and sample_weight must be tensors")
    if weight.dim() != 2 or weight.shape != sample_weight.shape:
        raise ValueError(f"kmeans_codebook: weight {tuple(weight.shape)} and sample_weight {tuple(sample_weight.shape)} "
                         "must be the same [out, in] shape")
    if not (weight.is_cuda and sample_weight.is_cuda) or weight.device != sample_weight.device:
        raise ValueError("kmeans_codebook: weight and sample_weight must be CUDA tensors on one device")
    if weight.shape[1] % 32:
        raise ValueError(f"kmeans_codebook: in_features={weight.shape[1]} must be a multiple of 32")
    w = weight.detach().float().contiguous()
    s = sample_weight.detach().float().contiguous()
    if not bool(torch.isfinite(w).all()):
        raise ValueError("kmeans_codebook: weight has non-finite values")
    if not bool((torch.isfinite(s) & (s >= 0)).all()):
        raise ValueError("kmeans_codebook: sample weights must be finite and >= 0")
    return quant_cuda.kmeans1d(w, s, 2 ** bits)


def _numpy_linear_quantile(sorted_flat, q):
    """numpy.quantile(..., method="linear") of a sorted 1-D fp32 tensor, as numpy evaluates it: the fraction and numpy's lerp
    (exact at both ends) in fp32.  -> 0-d fp32 tensor on the CPU."""
    n = sorted_flat.numel()
    h = (n - 1) * q
    lo = int(h // 1)
    t = torch.tensor(h - lo, dtype=torch.float32)
    a, b = sorted_flat[lo].cpu(), sorted_flat[min(lo + 1, n - 1)].cpu()
    diff = b - a
    return b - diff * (1 - t) if t >= 0.5 else a + diff * t


def outlier_threshold(weight, range):
    """The outlier threshold of generate_outlier_config.py:47-53: max(|q1 - r IQR|, |q3 + r IQR|) with numpy's
    linear-interpolation quartiles of all the layer's weights, r = `range`, evaluated in fp32 as numpy does for an fp32 array.
    Sorted on the tensor's device (torch.quantile rejects inputs of more than 2^24 elements)."""
    flat = torch.sort(weight.detach().float().reshape(-1)).values
    q1, q3 = _numpy_linear_quantile(flat, 0.25), _numpy_linear_quantile(flat, 0.75)
    lo, hi = q1 - range * (q3 - q1), q3 + range * (q3 - q1)
    return float(torch.maximum(lo.abs(), hi.abs()))


def split_outliers(weight, fisher, threshold=None, sensitivity=0.0):
    """-> (dense, outliers), both fp32 [out, in]: the masks of outliers.py.  Sensitivity first (outliers.py:14-23): the
    numel * sensitivity / 100 largest Fisher values by topk, then every weight whose Fisher value is STRICTLY above the last of
    them (ties with it stay dense; a count of 0 takes none).  Then the threshold on what remains (outliers.py:52-60):
    w >= threshold or w <= -threshold, in fp32."""
    w = weight.detach().float()
    mask = torch.zeros_like(w, dtype=torch.bool)
    if sensitivity:
        g = fisher.detach().to(w.device).float()
        if g.shape != w.shape:
            raise ValueError(f"split_outliers: fisher {tuple(g.shape)} must have the weight's shape {tuple(w.shape)}")
        num = int(g.numel() * sensitivity / 100)
        if num > 0:
            mask = g > g.reshape(-1).topk(k=num).values[-1]
    outliers = w * mask
    dense = w * ~mask
    if threshold is not None:
        t = torch.logical_or(dense >= threshold, dense <= -threshold)
        outliers = outliers + dense * t
        dense = dense * ~t
    return dense, outliers


def quantize_linear(linear, fisher, bits, threshold=None, sensitivity=0.0):
    """nn.Linear -> QuantLinearLUT on the linear's (CUDA) device, dense-and-sparse when a threshold or a sensitivity is given.

    Sample weight of each weight = fisher * (dense weight != 0); a row whose sum is 0 gets all ones (nuq.py:172-175).  The
    buffers are those QuantLinearLUT.pack2 makes from the same centroids, labels and outlier matrix: qweight packed on the device,
    the bias copied, CSR of (outlier - the row's centroid nearest to zero) (quant.py:117-123), topX = 0."""
    if bits not in (3, 4):
        raise ValueError(f"quantize_linear: bits={bits} must be 3 or 4")
    weight = linear.weight
    if not weight.is_cuda:
        raise ValueError("quantize_linear: the linear's weight must be on a CUDA device")
    out_f, in_f = weight.shape
    fisher = fisher.detach().to(weight.device).float()
    if fisher.shape != weight.shape:
        raise ValueError(f"quantize_linear: fisher {tuple(fisher.shape)} must have the weight's shape {tuple(weight.shape)}")
    sparse = threshold is not None or bool(sensitivity)
    if sparse:
        dense, outliers = split_outliers(weight, fisher, threshold, sensitivity)
    else:
        dense, outliers = weight.detach().float(), None
    lut, labels = kmeans_codebook(dense, fisher * (dense != 0), bits)

    buffers = {"qweight": quant_cuda.pack_indices(labels, bits), "lookup_table": lut,
               "bias": linear.bias.detach().clone() if linear.bias is not None else None}
    if sparse:
        zero = lut.gather(1, lut.abs().argmin(dim=1, keepdim=True))
        outliers = torch.where(outliers != 0, outliers - zero, outliers)
        csr = outliers.to_sparse(layout=torch.sparse_csr)
        buffers.update(rows=csr.crow_indices().to(torch.int32), cols=csr.col_indices().to(torch.int32),
                       vals=csr.values().to(torch.float32))
    return QuantLinearLUT.from_buffers(bits, buffers)


def _set_module(model, name, module):
    parent, _, attr = name.rpartition(".")
    setattr(model.get_submodule(parent) if parent else model, attr, module)


def quantize_model(model, fisher_state, bits, outlier_range=None, sensitivity=0.0, skip=("lm_head",)):
    """Replace every nn.Linear of `model` (checkpoint.find_linear_layers, except `skip`) by its quantize_linear result, in
    place and one layer at a time.  fisher_state[f"{name}.weight"] holds the layer's squared gradients (the reference's
    gradient checkpoints).  outlier_range: the IQR range of generate_outlier_config.py, giving each layer's threshold
    (outlier_threshold); sensitivity: the percentage of outliers.py.  Returns {layer name: CSR nnz} of the sparse layers;
    checkpoint.save_checkpoint(model, path, bits) then writes the reference's packed format."""
    layers = find_linear_layers(model)
    for name in skip:
        layers.pop(name, None)
    missing = [n for n in layers if f"{n}.weight" not in fisher_state]
    if missing:
        raise KeyError(f"quantize_model: fisher_state has no entry for {missing[:4]}{' ...' if len(missing) > 4 else ''}")
    numvals = {}
    for name, linear in layers.items():
        thr = outlier_threshold(linear.weight, outlier_range) if outlier_range is not None else None
        q = quantize_linear(linear, fisher_state[f"{name}.weight"], bits, threshold=thr, sensitivity=sensitivity)
        _set_module(model, name, q)
        if q.include_sparse:
            numvals[name] = q.numvals
        del linear
    return numvals


def dequantize_model(model, dtype=torch.float16):
    """The inverse of quantize_model: replace every QuantLinearLUT below `model` by its QuantLinearLUT.to_linear(dtype), in place
    and one layer at a time, after dissolving the sibling groups (fusion.fuse_siblings) of its layers.  model.state_dict() then
    has the keys of the dense model (`<layer>.weight`, `<layer>.bias`), so e.g. a Hugging Face model's save_pretrained writes a
    plain dense checkpoint.  Returns the names of the replaced layers."""
    layers = find_linear_layers(model, kinds=(QuantLinearLUT,))
    for q in layers.values():
        if q._sibling_group is not None:
            q._sibling_group[0].dissolve()
    names = list(layers)
    for name in names:
        _set_module(model, name, layers.pop(name).to_linear(dtype))
    return names


def fisher_information(model, batches, layers=None, skip=("lm_head",)):
    """The diagonal of the empirical Fisher information of the model's linear layers: {f"{name}.weight": fp32 [out, in]} with
    F = sum over every sequence s of every batch of g_s * g_s, g_s the layer's weight gradient of s's loss alone.  The result is
    the `fisher_state` of quantize_model.

    model: a Hugging Face causal LM in fp16 or bf16, called as model(ids).logits.  batches: an iterable of token tensors [B, T]
    (T >= 2), one sequence per row.  layers: names from checkpoint.find_linear_layers (not in `skip`) to restrict the result to -
    the fp32 result of a 7B model's decoder linears takes 25.9 GB, so a large model can be done in several passes; None: every
    linear not in `skip`.

    The loss of a sequence is the SUM of its next-token cross-entropies and a batch's loss is the sum over its sequences, so every
    g_s is the gradient of a batch holding s alone, and the batching changes F by rounding only.  (The sum also keeps the logit
    gradients O(1) rather than O(1/T), clear of fp16 underflow.)  F's scale does not matter to quantize_model: the weighted k-means
    and the sensitivity top-k are invariant to a constant factor.

    One backward per batch: forward hooks keep each selected layer's input x, a hook on its output receives dy, and
    quant_cuda.fisher_accumulate adds sum_s (dy_s^T x_s)^2 into F on the tensor cores, from the 16-bit x and dy, without forming
    any weight gradient.  No parameter requires grad during the run (the embedding's output does), so no .grad is created; the
    hooks, requires_grad and the training mode are restored afterwards, also on error.  Raises ValueError for a layer that runs
    more than once in one forward (tied or reused weights: its per-call squares would be wrong), is not fp16 / bf16, or has in or
    out features not a multiple of 8, and for a result that is not finite."""
    found = find_linear_layers(model)
    for name in skip:
        found.pop(name, None)
    if layers is not None:
        unknown = [n for n in layers if n not in found]
        if unknown:
            raise ValueError(f"fisher_information: layers {unknown[:4]} are not linear layers of the model outside skip={tuple(skip)}")
        found = {n: found[n] for n in layers}
    if not found:
        raise ValueError("fisher_information: no layer selected")
    for name, lin in found.items():
        if lin.weight.dtype not in _FISHER_DTYPES:
            raise ValueError(f"fisher_information: layer {name} is {lin.weight.dtype}; fp16 or bf16 is needed")
        if lin.in_features % 8 or lin.out_features % 8:
            raise ValueError(f"fisher_information: layer {name} is {lin.in_features} -> {lin.out_features}; in and out features must be "
                             "multiples of 8")
    fisher = {name: torch.zeros(lin.out_features, lin.in_features, device=lin.weight.device,
                                dtype=torch.promote_types(torch.float32, lin.weight.dtype)) for name, lin in found.items()}
    calls = dict.fromkeys(found, 0)
    seq_len = [0]

    def layer_hook(name):
        def hook(module, inputs, out):
            calls[name] += 1
            if calls[name] > 1:
                raise ValueError(f"fisher_information: layer {name} ran more than once in one forward (tied or reused weights)")
            x = inputs[0].detach()
            rows = x.numel() // module.in_features
            if rows % seq_len[0] or not out.requires_grad:
                raise ValueError(f"fisher_information: layer {name} did not see [B, T={seq_len[0]}, in] rows on the path to the loss")
            x = x.reshape(rows, module.in_features).contiguous()
            out.register_hook(lambda dy: quant_cuda.fisher_accumulate(
                x, dy.reshape(rows, module.out_features).contiguous(), fisher[name], seq_len[0]))
        return hook

    def embed_hook(module, inputs, out):
        return out.requires_grad_()

    saved = [(p, p.requires_grad) for p in model.parameters()]
    was_training = model.training
    handles = []
    try:
        for p, _ in saved:
            p.requires_grad_(False)
        model.eval()
        handles.append(model.get_input_embeddings().register_forward_hook(embed_hook))
        handles += [lin.register_forward_hook(layer_hook(name)) for name, lin in found.items()]
        for ids in batches:
            if ids.dim() != 2 or ids.shape[1] < 2:
                raise ValueError(f"fisher_information: a batch must be token ids [B, T] with T >= 2 (got {tuple(ids.shape)})")
            seq_len[0] = ids.shape[1]
            for name in calls:
                calls[name] = 0
            with torch.enable_grad():
                logits = model(ids).logits
                logits = logits[:, :-1].reshape(-1, logits.shape[-1])
                logits = logits.to(torch.promote_types(logits.dtype, torch.float32))  # fp32 softmax of 16-bit logits
                loss = torch.nn.functional.cross_entropy(logits, ids[:, 1:].reshape(-1), reduction="sum")
                del logits
                loss.backward()
    finally:
        for h in handles:
            h.remove()
        for p, rg in saved:
            p.requires_grad_(rg)
        model.train(was_training)
    for name, f in fisher.items():
        if not bool(torch.isfinite(f).all()):
            raise ValueError(f"fisher_information: the Fisher information of layer {name} is not finite")
    return {f"{name}.weight": f for name, f in fisher.items()}
