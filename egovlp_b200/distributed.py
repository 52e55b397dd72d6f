"""Data-parallel plumbing of the step: the embedding / tag all-gather with the reference's local-slice backward,
packed into ONE collective, and the fused training step.

Reference semantics (trainer/trainer_egoclip.py:11-27, 125-135): every rank gathers video/text embeddings and
verb/noun tag vectors, computes the full [G, G] loss redundantly, and back-propagates only its own B rows (no
reduce-scatter); DDP then averages parameter gradients, so the effective gradient is grad(global loss)/world.
"""
import torch
import torch.distributed as dist


def _world():
    if dist.is_available() and dist.is_initialized():
        return dist.get_world_size(), dist.get_rank()
    return 1, 0


def _all_gather_rows(t):
    """[B, C] -> [world*B, C], rank-major (== torch.cat(all_gather(list), 0) of the reference)."""
    world, _ = _world()
    if world == 1:
        return t
    t = t.contiguous()
    out = torch.empty((world * t.shape[0],) + tuple(t.shape[1:]), dtype=t.dtype, device=t.device)
    try:
        dist.all_gather_into_tensor(out, t)
    except (RuntimeError, NotImplementedError):   # backends without the flat variant
        parts = [torch.empty_like(t) for _ in range(world)]
        dist.all_gather(parts, t)
        out = torch.cat(parts, 0)
    return out


class AllGatherLocalGrad(torch.autograd.Function):
    """AllGather_multi of the reference trainers: forward all_gather + cat; backward keeps ONLY this rank's slice."""

    @staticmethod
    def forward(ctx, tensor):
        ctx.batch = tensor.shape[0]
        return _all_gather_rows(tensor)

    @staticmethod
    def backward(ctx, grad_output):
        _, rank = _world()
        return grad_output[ctx.batch * rank: ctx.batch * (rank + 1)]


class PackedGather(torch.autograd.Function):
    """One collective for (text, video, verb, noun): rows are packed as [text | video | verb | noun] fp32 and
    gathered with a single ncclAllGather; backward returns the local slices of the text / video gradients."""

    @staticmethod
    def forward(ctx, text, video, verb, noun):
        world, _ = _world()
        ctx.batch, ctx.ct, ctx.cv = text.shape[0], text.shape[1], video.shape[1]
        if world == 1:
            return text, video, verb, noun
        packed = torch.cat([text.float(), video.float(), verb.float(), noun.float()], dim=1)
        g = _all_gather_rows(packed)
        c0, c1, c2 = ctx.ct, ctx.ct + ctx.cv, ctx.ct + ctx.cv + verb.shape[1]
        return g[:, :c0].contiguous(), g[:, c0:c1].contiguous(), g[:, c1:c2].contiguous(), g[:, c2:].contiguous()

    @staticmethod
    def backward(ctx, gt, gv, _gverb, _gnoun):
        _, rank = _world()
        sl = slice(ctx.batch * rank, ctx.batch * (rank + 1))
        return gt[sl], gv[sl], None, None


def egoclip_step_loss(model, loss_fn, data):
    """Forward of one EgoClip pretraining step, fused: model -> ONE packed gather -> ONE fused similarity + EgoNCE
    kernel reading the gathered buffer in place (positives from bit-packed tags), whose backward kernel emits the local
    gradient slice.  Equivalent to trainer/trainer_egoclip.py:125-135."""
    text_embeds, video_embeds = model(data)
    world, rank = _world()
    loss = loss_fn.gathered(text_embeds, video_embeds, data["verb_vec"], data["noun_vec"], _all_gather_rows, rank, world)
    if loss is not None:
        return loss
    # G > 512 (more than 8 ranks x 64 clips): packed gather + the kernel-per-stage loss path
    t, v, verb, noun = PackedGather.apply(text_embeds, video_embeds, data["verb_vec"], data["noun_vec"])
    return loss_fn.fused(t, v, verb, noun)
