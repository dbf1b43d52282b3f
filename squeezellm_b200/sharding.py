"""Column sharding of a QuantLinearLUT across GPUs (BASELINE.json north_star; SURVEY.md section 8(e)).

The reference has no multi-GPU code at all.  Output channels are independent: column c of `qweight`, row c of
`lookup_table`, CSR row c and the dense-row entries whose `full_row_indices` equal c are all that y[c] needs (plus the
whole x).  Rank r of P therefore owns a contiguous range of output channels [c0, c1):

    qweight[:, c0:c1]   lookup_table[c0:c1]   rows[c0:c1+1] - rows[c0], cols/vals[rows[c0]:rows[c1]]
    full_rows[:, j], full_row_indices[j] - c0   for the j with c0 <= full_row_indices[j] < c1     (others dropped)

and computes its slice of y with the ordinary single-GPU kernel; the full output vector is the sum of the
zero-padded slices - ONE all-reduce (sum) on the output vector, as north_star specifies.  Ranges are cut on multiples
of 4 channels (the kernel's only width requirement; the reference kernel would need multiples of 128, which 22016/8
cannot give - SURVEY.md 8(e)).

`shard_bounds`, `shard_state` are pure functions on CPU tensors (testable with gloo); `ShardedQuantLinearLUT` is the
module that runs the local shard on its GPU and all-reduces.  `matvec_fn` lets tests substitute the CPU oracle for the
local compute - the product path always uses the CUDA module.
"""
import torch
import torch.nn as nn

from .fusion import SiblingGroup, stack_buffers
from .quant import QuantLinearLUT


def shard_bounds(outfeatures, world, align=4):
    """Contiguous, `align`-aligned, as-equal-as-possible output ranges: list of (c0, c1), len == world."""
    assert outfeatures % align == 0, f"outfeatures={outfeatures} must be a multiple of {align}"
    units = outfeatures // align
    base, extra = divmod(units, world)
    bounds, c = [], 0
    for r in range(world):
        n = (base + (1 if r < extra else 0)) * align
        bounds.append((c, c + n))
        c += n
    assert c == outfeatures
    return bounds


def shard_state(state, c0, c1):
    """Slice a QuantLinearLUT state dict (reference buffer names, squeezellm/quant.py:48-95) to channels [c0, c1).  Every tensor
    of the result is a contiguous copy of its own, in the dtype of the layer's buffer (int32 indices, fp32 values), as
    load_state_dict into a fresh layer would give it: a shard keeps no view of the full layer's storage."""
    out = {"qweight": state["qweight"][:, c0:c1], "lookup_table": state["lookup_table"][c0:c1]}
    if state.get("bias") is not None:
        out["bias"] = state["bias"][c0:c1]
    if state.get("rows") is not None:
        rows = state["rows"]
        a, b = int(rows[c0]), int(rows[c1])
        out["rows"] = rows[c0:c1 + 1] - rows[c0]
        out["cols"] = state["cols"][a:b]
        out["vals"] = state["vals"][a:b]
    if state.get("full_rows") is not None:
        idx = state["full_row_indices"]
        keep = torch.nonzero((idx >= c0) & (idx < c1)).flatten()
        # keep the dense-row count fixed across ranks (buffers of identical shape): dropped columns become zero columns
        fr = torch.zeros_like(state["full_rows"])
        fi = torch.zeros_like(idx)
        fr[:, :len(keep)] = state["full_rows"][:, keep]
        fi[:len(keep)] = (idx[keep] - c0).to(idx.dtype)
        out["full_rows"], out["full_row_indices"] = fr, fi
    return {k: v.to(torch.float32 if v.is_floating_point() else torch.int32, memory_format=torch.contiguous_format, copy=True)
            for k, v in out.items()}


class ShardedQuantLinearLUT(nn.Module):
    """One rank's column shard of a QuantLinearLUT + the all-reduce that rebuilds the full output vector.  Gives no gradient:
    its output is built in place by the all-reduce, outside autograd."""

    def __init__(self, local, outfeatures, c0, c1, group=None, matvec_fn=None):
        super().__init__()
        self.local = local                  # QuantLinearLUT over channels [c0, c1)  (or None when matvec_fn is given)
        self.outfeatures, self.c0, self.c1, self.group = outfeatures, c0, c1, group
        self.matvec_fn = matvec_fn          # tests: CPU stand-in for the local compute

    @classmethod
    def from_full(cls, full_state, bits, infeatures, outfeatures, rank, world, include_sparse, topX, device, group=None):
        """Rank `rank`'s shard of the layer whose state dict is `full_state` (QuantLinearLUT.from_buffers on shard_state).
        `infeatures`, `include_sparse` and `topX` must be those of full_state's buffers (CSR arrays: include_sparse)."""
        c0, c1 = shard_bounds(outfeatures, world)[rank]
        m = QuantLinearLUT.from_buffers(bits, shard_state(full_state, c0, c1))
        if (m.infeatures, m.include_sparse, m.topX) != (infeatures, bool(include_sparse), topX):
            raise ValueError(f"ShardedQuantLinearLUT.from_full: full_state holds a layer with in_features={m.infeatures}, "
                             f"include_sparse={m.include_sparse}, topX={m.topX}; the arguments say {infeatures}, "
                             f"{bool(include_sparse)}, {topX}")
        return cls(m.to(device), outfeatures, c0, c1, group)

    def forward(self, x):
        import torch.distributed as dist
        # _forward_impl: no autograd node here - the in-place all-reduce below carries no gradient
        y_local = self.matvec_fn(x) if self.matvec_fn is not None else self.local._forward_impl(x)
        lead = y_local.shape[:-1]
        full = torch.zeros(lead + (self.outfeatures,), dtype=y_local.dtype, device=y_local.device)
        full[..., self.c0:self.c1] = y_local
        dist.all_reduce(full, op=dist.ReduceOp.SUM, group=self.group)  # sum of zero-padded slices
        return full


def exchange_stacked(y_local, members, rank, world, out=None, group=None):
    """Rebuild the full outputs of `members` sibling layers from one rank's stacked shard result.

    y_local [..., members*w] is what this rank's stacked shard (fusion.SiblingGroup over its column shards, all of width
    w = N/world) produced: member m's channels [rank*w, (rank+1)*w) at [m*w, (m+1)*w).  They are placed into a zeroed
    [..., members, N] buffer and summed over ranks with ONE all-reduce (north_star's exchange, once per stacked launch
    instead of once per member).  Returns that buffer; [..., m, :] is member m's full output vector.
    `out` (optional, [..., members, N], same dtype/device) is reused instead of allocating."""
    import torch.distributed as dist
    lead = y_local.shape[:-1]
    w = y_local.shape[-1] // members
    if out is None:
        out = torch.zeros(lead + (members, w * world), dtype=y_local.dtype, device=y_local.device)
    else:
        out.zero_()
    out.view(lead + (members, world, w))[..., rank, :] = y_local.reshape(lead + (members, w))
    dist.all_reduce(out, op=dist.ReduceOp.SUM, group=group)
    return out


class PeerExchange:
    """Arena in torch symmetric memory (peer-mapped over NVLink) + the bookkeeping `quant_cuda.lutgemv_fused_exchange`
    needs: the kernel's finishing CTAs store their slice of y into every rank's arena and wait for the peers', so a
    column-sharded layer needs no separate collective (include/sqllm_b200.h, sqllm_lutgemv_fused_exchange).  Its results
    carry no gradient.

    One arena per rank, identical layout everywhere: [0,8) arrival counter, [64,72) expected arrivals (local), [128,132)
    error word, destination vectors from 4096 on (one per `name`, [members][out_features_full] in the activation dtype).
    Consecutive exchanges must use different names (a fast rank may deliver the next result while a slow one still reads
    the previous one).  All ranks must call `forward` in the same order."""

    FLAG, STATE, ERROR, DATA = 0, 64, 128, 4096

    def __init__(self, rank, world, device, arena_bytes=8 << 20, group=None):
        """Collective: every rank of `group` must construct its PeerExchange at the same point (ends with a barrier)."""
        import torch.distributed as dist
        import torch.distributed._symmetric_memory as symm
        self.rank, self.world, self.device = rank, world, device
        self.group = group if group is not None else dist.group.WORLD
        self.arena = symm.empty(arena_bytes, dtype=torch.uint8, device=device)
        self.hdl = symm.rendezvous(self.arena, self.group)
        self.arena.zero_()
        torch.cuda.synchronize(device)
        dist.barrier(group=self.group)          # every arena is zeroed before anybody's kernel can touch it
        self.peer_base = int(self.hdl.buffer_ptrs_dev)
        self.offsets, self.next = {}, self.DATA
        self.arena_bytes = arena_bytes
        self.calls, self.check_every = 0, 4096   # forward() polls the error word every check_every calls (0 = never; check() is public)

    def _slot(self, name, members, n_full, dtype):
        key = (name, members, n_full, dtype)
        if key not in self.offsets:
            nbytes = members * n_full * torch.empty(0, dtype=dtype).element_size()
            off = self.next
            self.next = (off + nbytes + 255) & ~255
            if self.next > self.arena_bytes:
                raise RuntimeError("PeerExchange arena exhausted")
            view = self.arena[off:off + nbytes].view(dtype).view(members, n_full)
            self.offsets[key] = (off, view)
        return self.offsets[key]

    def forward(self, layer, x, name, members, n_full):
        """Run `layer` (this rank's column shard, possibly a stacked sibling group's layer) on x; returns the local
        [members, n_full] vector holding every rank's slices once the launch has completed (stream order)."""
        from .quant import quant_cuda
        off, view = self._slot(name, members, n_full, x.dtype)
        self.calls += 1
        if self.check_every and self.calls % self.check_every == 0 and not torch.cuda.is_current_stream_capturing():
            self.check()  # surfaces a timed-out wait in the product path (costs a device synchronisation: every check_every calls only)
        rows, cols, vals, fr, fri = layer._sparse_args()
        # bf16 x has a binding of its own (bf16 vectors in the arenas); fp16 / fp32 x keep theirs
        call = quant_cuda.lutgemv_fused_exchange_bf16 if x.dtype == torch.bfloat16 else quant_cuda.lutgemv_fused_exchange
        call(x.contiguous().reshape(-1), layer.qweight, layer.lookup_table, layer.bits, layer.bias, rows, cols, vals, fr, fri,
             self.peer_base, off, self.FLAG, self.STATE, self.ERROR, self.world, self.rank, members, n_full)
        return view

    def error(self):
        """True if some wait inside a kernel timed out (a peer never delivered).  Synchronises the device."""
        return bool(self.arena[self.ERROR:self.ERROR + 4].view(torch.int32).item())

    def check(self):
        """Raise if the error word is set: after a timeout the vector that call delivered is incomplete and every later wait is
        skipped (the kernel does not block on a dead peer twice), so results from that point on are not valid."""
        if self.error():
            raise RuntimeError("PeerExchange: an in-kernel wait for a peer rank timed out (2 s); results since then are incomplete. "
                               "Call resync() on every rank once all ranks are alive again.")

    def resync(self):
        """Collective: bring every rank's counters back to a common, clean state after a timeout (or at any quiescent point).
        All ranks must call it with no exchange launch in flight."""
        import torch.distributed as dist
        torch.cuda.synchronize(self.device)
        dist.barrier(group=self.group)
        self.arena[:self.DATA].zero_()
        torch.cuda.synchronize(self.device)
        dist.barrier(group=self.group)



class PeerArena:
    """Peer-visible arenas for `runtime.DecodeSequence` on several GPUs (one process per GPU).

    The sequence kernel hands the result of one matvec to the next as self-validating tagged words in an arena
    (csrc/lutgemv_seq.cuh); on several GPUs the owner of a strip stores its words into EVERY rank's arena over NVLink, and the
    next matvec's input poll is the whole exchange - no collective, no flag.  `arena_for` is collective (symmetric-memory
    rendezvous + barrier): every rank must compile its sequences in the same order."""

    def __init__(self, rank, world, device, group=None):
        import torch.distributed as dist
        self.rank, self.world, self.device = rank, world, torch.device(device)
        self.group = group if group is not None else dist.group.WORLD
        self._keep = []

    def arena_for(self, nbytes):
        import torch.distributed as dist
        import torch.distributed._symmetric_memory as symm
        nbytes = (int(nbytes) + 4095) // 4096 * 4096
        arena = symm.empty(nbytes, dtype=torch.uint8, device=self.device)
        hdl = symm.rendezvous(arena, self.group)
        arena.zero_()
        torch.cuda.synchronize(self.device)
        dist.barrier(group=self.group)   # every arena is zeroed before any rank's kernel can store into it
        self._keep.append((arena, hdl))
        return arena, int(hdl.buffer_ptrs_dev)


class ShardedSiblingGroup(SiblingGroup):
    """Column shards of a set of sibling layers (same input) run as ONE stacked launch per rank + ONE exchange.  Gives no
    gradient: the exchange runs outside autograd.

    Built from the full (unsharded) QuantLinearLUT members: every rank keeps columns [rank*w, (rank+1)*w) of each member
    (`shard_state`), stacks those shards along N (`fusion.stack_buffers`) and answers the members' `forward(x)` through
    `fusion.SiblingGroup`'s one-result cache - so model code is unchanged: `q_proj(x)`, `k_proj(x)`, `v_proj(x)` return
    FULL-width vectors on every rank.  The exchange is `PeerExchange` (in-kernel stores over NVLink, no collective) when one is
    given, else one NCCL all-reduce per stacked launch (`exchange_stacked`).
    A single layer (o_proj, down_proj) is simply a group of one.  `compute` lets CPU tests stand in for the CUDA launch."""

    def __init__(self, members, rank, world, name, peer=None, group=None, compute=None):
        self.members, self.rank, self.world, self.name, self.peer, self.pg, self.compute = list(members), rank, world, name, peer, group, compute
        n_full = {m.outfeatures for m in self.members}
        if len(n_full) != 1:
            raise ValueError("sibling layers sharded together must have the same out_features")
        self.n_full = n_full.pop()
        c0, c1 = shard_bounds(self.n_full, world)[rank]
        if (c1 - c0) * world != self.n_full:
            raise ValueError(f"out_features={self.n_full} does not split into {world} equal 4-aligned shards")
        self.w = c1 - c0
        shards = [QuantLinearLUT.from_buffers(m.bits, shard_state(m.state_dict(), c0, c1)) for m in self.members]
        self._join(stack_buffers(shards))
        layer = self.layer
        for m, o in zip(self.members, self.offsets):
            # the member keeps its buffer names but now holds this rank's shard (views of the stacked storage)
            m.qweight = layer.qweight[:, o:o + self.w]
            m.lookup_table = layer.lookup_table[o:o + self.w]
            for k in ("rows", "cols", "vals", "full_rows", "full_row_indices"):
                if hasattr(m, k):
                    delattr(m, k)
            m.include_sparse, m.numvals, m.topX = False, 0, 0
            if m.bias is not None:
                m.bias = layer.bias[o:o + self.w]

    def member_columns(self, i):
        raise NotImplementedError("QuantLinearLUT.dequantize: this layer is column-sharded (sharding.shard_model) and holds only "
                                  "this rank's columns; dequantize the full layer before sharding it")

    def dissolve(self):
        raise NotImplementedError("ShardedSiblingGroup.dissolve: its members hold only this rank's columns and cannot stand "
                                  "alone again; rebuild the full layers from the checkpoint instead")

    def _stacked(self, x):
        nm = len(self.members)
        if self.compute is not None:
            y = self.compute(self.layer, x)
        elif self.peer is not None and x.shape[-1] == x.numel():
            return self.peer.forward(self.layer, x, self.name, nm, self.n_full)       # [members, n_full], exchange done in-kernel
        else:
            y = self.layer._forward_impl(x)  # no autograd node: the exchange carries no gradient
        return exchange_stacked(y, nm, self.rank, self.world, group=self.pg)            # [..., members, n_full]

    def _member_result(self, i, x, y):
        y = y[..., i, :]
        if self.peer is not None and self.compute is None:
            # the peer path returns a view of a persistent arena slot that the next call of this layer overwrites (remotely, from
            # other ranks): hand out a private copy, like nn.Linear would (N elements - nothing next to the matvec)
            y = y.clone()
        if y.dim() < x.dim():                      # decode-shaped input [1, 1, K] -> [1, 1, N] like QuantLinearLUT.forward
            y = y.reshape(x.shape[:-1] + (self.n_full,))
        return y


def shard_model(model, rank, world, peer=None, group=None, siblings=(("q_proj", "k_proj", "v_proj"), ("gate_proj", "up_proj"))):
    """Column-shard every QuantLinearLUT of `model` in place for rank `rank` of `world`: sibling sets become one
    ShardedSiblingGroup each, every other QuantLinearLUT a group of one.  Every rank must call it on the same model.
    Returns the groups (their `.launches` count stacked launches).  Exchange names alternate so that consecutive launches
    never share a destination (PeerExchange's requirement)."""
    groups = []
    for mod_name, mod in model.named_modules():
        taken = set()
        for names in siblings:
            ms = [getattr(mod, n, None) for n in names]
            if all(isinstance(m, QuantLinearLUT) and m._sibling_group is None for m in ms) and len({m.outfeatures for m in ms}) == 1:
                groups.append(ShardedSiblingGroup(ms, rank, world, f"{mod_name}.{'+'.join(names)}", peer=peer, group=group))
                taken.update(names)
        for n, child in mod.named_children():
            if isinstance(child, QuantLinearLUT) and n not in taken and child._sibling_group is None:
                groups.append(ShardedSiblingGroup([child], rank, world, f"{mod_name}.{n}", peer=peer, group=group))
    if world > 1:
        import torch.distributed as dist
        if dist.is_available() and dist.is_initialized():
            # ranks finish the CPU-side sharding at different times; the in-kernel waits are bounded (2 s), so nobody may start
            # exchanging before everybody is ready
            if torch.cuda.is_available():
                torch.cuda.synchronize()
            dist.barrier(group=group)
    return groups
