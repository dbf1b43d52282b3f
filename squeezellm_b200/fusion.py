"""Sibling fusion: QuantLinearLUT layers that read the same input run as ONE launch.

The reference issues one kernel sequence per nn.Linear replacement (squeezellm/quant.py:211-312); in a LLaMA decoder
q_proj/k_proj/v_proj read the same hidden state and so do gate_proj/up_proj (the call sites are in transformers'
LlamaAttention / LlamaMLP, which llama.py drives).  Stacking their packed matrices along the output dimension turns three
(two) batch-1 matvecs into one matvec of 3x (2x) the width: same arithmetic per output channel, bit-identical packed
indices and LUT rows, 224 -> 128 launches per LLaMA-7B token.

Nothing in the model code changes.  `fuse_siblings(model)` concatenates the members' buffers
    qweight [K/32*bits, N_i] -> [K/32*bits, sum N_i]     lookup_table [N_i, 2^bits] -> [sum N_i, 2^bits]
    rows/cols/vals (CSR by output channel) -> one CSR    full_rows [K, topX_i] -> [K, sum topX_i]  (+ shifted indices)
into a hidden QuantLinearLUT and re-points every member's buffers at views of it (no second copy of the weights stays
alive).  A member's forward(x) then asks the group: the first sibling called with a given x runs the stacked layer, the
others return their slice of that result.  The cache key is the identity of the input tensor object plus its in-place
version counter, each member may consume a result once, and the reference to x is dropped when all members have consumed
it - a call pattern that does not share x simply recomputes (correct, just not faster).
"""
import torch

from .quant import QuantLinearLUT

__all__ = ["SiblingGroup", "fuse_siblings", "LLAMA_SIBLINGS"]

LLAMA_SIBLINGS = (("q_proj", "k_proj", "v_proj"), ("gate_proj", "up_proj"))


def _version(x):
    try:
        return x._version
    except RuntimeError:  # inference-mode tensors carry no version counter
        return -1


def stack_buffers(members):
    """Concatenate the buffer sets of `members` along the output dimension.  Pure tensor code (runs on any device);
    returns the kwargs/buffers of the stacked layer.  Exposed for the CPU tests."""
    m0 = members[0]
    K, bits = m0.infeatures, m0.bits
    dev = m0.qweight.device
    for m in members:
        if m.infeatures != K or m.bits != bits or m.qweight.device != dev:
            raise ValueError("siblings must share in_features, bits and device")
    n_out = [m.outfeatures for m in members]
    offs = [0]
    for n in n_out:
        offs.append(offs[-1] + n)
    out = {"offsets": offs, "bits": bits, "infeatures": K, "outfeatures": offs[-1]}
    out["qweight"] = torch.cat([m.qweight for m in members], dim=1).contiguous()
    out["lookup_table"] = torch.cat([m.lookup_table for m in members], dim=0).contiguous()
    if any(m.bias is not None for m in members):
        out["bias"] = torch.cat([m.bias.float() if m.bias is not None else torch.zeros(m.outfeatures, device=dev)
                                 for m in members]).contiguous()
    else:
        out["bias"] = None
    # each member's outliers as its own forward reads them, so that its slice of the stacked result is what it gives alone
    sparse = [m._sparse_args() for m in members]
    if any(s[0] is not None for s in sparse):
        rows, cols, vals, base = [torch.zeros(1, dtype=torch.int32, device=dev)], [], [], 0
        for m, (r, c, v, _, _) in zip(members, sparse):
            if r is not None:
                r = r.to(torch.int64)
                rows.append((r[1:] + base).to(torch.int32))
                cols.append(c)
                vals.append(v)
                base += int(r[-1])
            else:
                rows.append(torch.full((m.outfeatures,), base, dtype=torch.int32, device=dev))
        out["rows"] = torch.cat(rows).contiguous()
        out["cols"] = torch.cat(cols).contiguous() if cols else torch.zeros(0, dtype=torch.int32, device=dev)
        out["vals"] = torch.cat(vals).contiguous() if vals else torch.zeros(0, dtype=torch.float32, device=dev)
    dense = [(s[3], s[4] + o) for s, o in zip(sparse, offs) if s[3] is not None]
    if dense:
        out["full_rows"] = torch.cat([fr for fr, _ in dense], dim=1).contiguous()
        out["full_row_indices"] = torch.cat([fri for _, fri in dense]).to(torch.int32).contiguous()
    return out


class SiblingGroup:
    """The stacked layer of a set of sibling QuantLinearLUT modules plus the one-result cache described above."""

    def __init__(self, members, share_storage=True):
        self.members = list(members)
        self._join(stack_buffers(self.members))
        if share_storage:  # members keep their buffer names (state_dict stays loadable/savable) as views of the stacked storage
            for m, o in zip(self.members, self.offsets):
                m.qweight = self.layer.qweight[:, o:o + m.outfeatures]
                m.lookup_table = self.layer.lookup_table[o:o + m.outfeatures]

    def _join(self, stacked):
        """Make the stacked layer from stack_buffers' result and hand every member's forward to this group, with an empty cache."""
        self.offsets = stacked["offsets"]
        self.layer = QuantLinearLUT.from_buffers(stacked["bits"], stacked)
        for i, m in enumerate(self.members):
            object.__setattr__(m, "_sibling_group", (self, i))
        self._x = self._ver = self._y = None
        self._pending = set()
        self.launches = 0  # stacked launches issued (tests / bench count these)

    def member_forward(self, i, x):
        if not (self._x is x and self._ver == _version(x) and i in self._pending):
            self._y = self._stacked(x)
            self._x, self._ver = x, _version(x)
            self._pending = set(range(len(self.members)))
            self.launches += 1
        self._pending.discard(i)
        y = self._member_result(i, x, self._y)
        if not self._pending:
            self._x = self._y = None
        return y

    def _stacked(self, x):
        """The stacked result for x, computed once per input and shared by the members."""
        return self.layer(x)

    def _member_result(self, i, x, y):
        """Member i's output out of the stacked result y."""
        y = y[..., self.offsets[i]:self.offsets[i + 1]]
        if y.dtype != x.dtype and self.members[i].bias is None:
            # another member's bias promoted the stacked batch result to fp32 (out.to(dtype) + fp32 bias); this member has none, so
            # its slice is its x-dtype output + 0.0: casting back is exact and gives the dtype and bits it returns alone
            y = y.to(x.dtype)
        return y

    def member_columns(self, i):
        """(stacked layer, first column) of member i's weights: what QuantLinearLUT.dequantize reads."""
        return self.layer, self.offsets[i]

    def dissolve(self):
        """Make every member a stand-alone layer again: buffers that are views of the stacked layer become the member's own
        contiguous copies, and the member forgets the group (its forward then runs its own buffers)."""
        for m in self.members:
            for name in ("qweight", "lookup_table"):
                t = getattr(m, name)
                if t._base is not None:  # a view of the stacked buffer (share_storage)
                    setattr(m, name, t.clone(memory_format=torch.contiguous_format))
            object.__setattr__(m, "_sibling_group", None)
        self._x = self._y = None
        self._pending = set()


def fuse_siblings(model, groups=LLAMA_SIBLINGS, share_storage=True):
    """Group sibling QuantLinearLUT attributes of every sub-module of `model` (default: LLaMA's q/k/v and gate/up).
    Call it after the checkpoint is loaded and the model is on its device.  Groups with a member whose codebook is being trained
    (QuantLinearLUT.train_codebook) are left unfused.  Returns the SiblingGroup list."""
    made = []
    for mod in model.modules():
        for names in groups:
            ms = [getattr(mod, n, None) for n in names]
            if not all(isinstance(m, QuantLinearLUT) for m in ms):
                continue
            if any(getattr(m, "_sibling_group", None) is not None for m in ms):
                continue
            if len({(m.infeatures, m.bits, m.qweight.device) for m in ms}) != 1:
                continue
            if any(m._trained for m in ms):  # codebook training (QuantLinearLUT.train_codebook) runs on unstacked layers only
                continue
            made.append(SiblingGroup(ms, share_storage=share_storage))
    return made
