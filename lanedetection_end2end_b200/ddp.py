"""Data-parallel plumbing (new capability -- the reference is single-GPU, SURVEY.md 2.1/8e):
one process per GPU, full model replica, per-replica BatchNorm statistics, and ONE
all-reduce (sum, then 1/world) over a single flat fp32 gradient buffer per step
(2 063 344 elements = 8.25 MB for the 2-lane model).  Parameters whose gradient is None
(``net.encoder.output_conv``, unused in training -- BP/Networks/ERFNet.py:84,92-93)
contribute zeros so every rank reduces the same layout.
"""
import torch
import torch.distributed as dist


class FlatGradAllReduce:
    def __init__(self, module, process_group=None):
        self.params = [p for p in module.parameters() if p.requires_grad]
        self.group = process_group
        self.numel = sum(p.numel() for p in self.params)
        p0 = self.params[0]
        self.flat = torch.zeros(self.numel, dtype=torch.float32, device=p0.device)
        self.views = []
        off = 0
        for p in self.params:
            self.views.append(self.flat[off:off + p.numel()].view_as(p))
            off += p.numel()

    def attach(self):
        """Make every existing ``p.grad`` a view into the flat buffer (like DDP's gradient_as_bucket_view): backward then
        accumulates straight into the buffer and a step needs no pack / unpack copies at all.  Call after a backward
        (so the gradients exist) and keep the gradients alive (zero them in place, never ``set_to_none``)."""
        self.flat.zero_()
        for p, v in zip(self.params, self.views):
            if p.grad is not None:
                v.copy_(p.grad)
                p.grad = v
        self.attached = True

    def _is_attached(self):
        return getattr(self, "attached", False) and all(
            p.grad is None or p.grad.data_ptr() == v.data_ptr() for p, v in zip(self.params, self.views))

    def pack(self):
        have = [(v, p.grad) for p, v in zip(self.params, self.views) if p.grad is not None]
        for p, v in zip(self.params, self.views):
            if p.grad is None:
                v.zero_()
        if have:
            torch._foreach_copy_([v for v, _ in have], [g for _, g in have])     # one fused launch

    def unpack(self):
        have = [(p.grad, v) for p, v in zip(self.params, self.views) if p.grad is not None]
        if have:
            torch._foreach_copy_([g for g, _ in have], [v for _, v in have])

    def __call__(self):
        """Average gradients over the group; returns the flat buffer (for tests)."""
        world = dist.get_world_size(self.group) if dist.is_initialized() else 1
        attached = self._is_attached()
        if not attached:
            self.pack()
        if world > 1:
            dist.all_reduce(self.flat, op=dist.ReduceOp.SUM, group=self.group)
            self.flat.mul_(1.0 / world)
        if not attached:
            self.unpack()
        return self.flat


def any_rank_nonzero(word, out, group=None):
    """out[0] = max over the group's ranks of word[0] (int32 status words, >= 0): nonzero iff any rank's word is nonzero.
    The guarded optimizer update reads it, so that a singular system on one rank skips the update on every rank and the
    replicas, which apply the same averaged gradients, stay identical.  One capturable all-reduce of one element."""
    out.copy_(word)
    if dist.is_initialized() and dist.get_world_size(group) > 1:
        dist.all_reduce(out, op=dist.ReduceOp.MAX, group=group)
    return out


def broadcast_parameters(module, src=0, group=None):
    """Make every replica start from rank ``src``'s parameters and buffers."""
    if not dist.is_initialized() or dist.get_world_size(group) == 1:
        return
    for t in list(module.parameters()) + list(module.buffers()):
        dist.broadcast(t.data, src, group=group)


def lane_valid_scale(valid, nlanes, group=None):
    """Per-lane factors that turn DDP's "mean of per-shard losses" into the reference's batch-global normaliser.

    ``backprojection_loss`` divides the squared error of lane l by the number of valid samples of lane l in the WHOLE batch
    (BP/Loss_crit.py:215).  With the batch sharded over R ranks each shard divides by its own count n_r; multiplying the
    shard's lane loss by  f = R * n_r / sum_r n_r  (one all-reduce of `nlanes` scalars) makes the rank-mean of the losses --
    and of every gradient, which the flat all-reduce averages -- identical to the single-process big-batch value
    (SURVEY.md 8e "subtlety").  valid: [B, >= nlanes, 56]; returns float64 [nlanes] on valid's device.  Pass it as
    ``lane_scale`` to Loss_crit.fused_backprojection_loss / backprojection_loss.forward_lanes."""
    local = valid[:, :nlanes].double().sum(dim=(0, 2))
    if not dist.is_initialized() or dist.get_world_size(group) == 1:
        return torch.ones_like(local)
    total = local.clone()
    dist.all_reduce(total, op=dist.ReduceOp.SUM, group=group)
    world = dist.get_world_size(group)
    return torch.where(total == 0, torch.ones_like(total), world * local / torch.where(total == 0, torch.ones_like(total), total))
