"""Losses of the reference's model/loss.py on CUDA kernels: same class names, constructor arguments and
forward signatures -- the contrastive losses of pretraining / EPIC-MIR and the CrossEntropy of the Ego4D OSCC / PNR
fine-tuning heads."""
import torch
from torch import nn

from .. import engine, ops


class NormSoftmaxLoss(nn.Module):
    def __init__(self, temperature=0.05):
        super().__init__()
        self.temperature = temperature

    def forward(self, x):
        G = x.shape[0]
        if x.dim() != 2 or x.shape[1] != G:
            raise NotImplementedError(f"NormSoftmaxLoss: square similarity matrix expected, got {tuple(x.shape)}")
        mask = ops.positives_mask_from_sims(None, None, G, 0, device=x.device)
        return engine.NceLossFn.apply(x, mask, self.temperature)


class EgoNCE(nn.Module):
    def __init__(self, temperature=0.05, noun=True, verb=True):
        super().__init__()
        self.noun, self.verb, self.temperature = noun, verb, temperature

    def _mode(self):
        return 1 if (self.noun and self.verb) else 2 if self.noun else 3

    def forward(self, x, mask_v, mask_n):
        """x, mask_v (= sim_matrix(verb, verb)), mask_n (= sim_matrix(noun, noun)): [G, G] float, as the
        unchanged trainer passes them (trainer/trainer_egoclip.py:132-135)."""
        G = x.shape[0]
        mask = ops.positives_mask_from_sims(mask_v.detach().contiguous().float(), mask_n.detach().contiguous().float(),
                                            G, self._mode())
        return engine.NceLossFn.apply(x, mask, self.temperature)

    def fused(self, text_embeds, video_embeds, verb_vec, noun_vec):
        """Fused entry: gathered embeddings + multi-hot tags -> loss, without materialising the
        verb/noun similarity matrices (positives from bit-packed tag co-occurrence)."""
        G, Cc = text_embeds.shape
        if ops.egonce_fused_supported(G, Cc) and video_embeds.shape[1] == Cc:      # ONE kernel per direction
            f = lambda t: t if (t.dtype == torch.float32 and t.stride(1) == 1) else t.float().contiguous()
            mode = self._mode()
            return engine.FusedEgoNceFn.apply(f(text_embeds), f(video_embeds), f(verb_vec) if mode in (1, 3) else None,
                                              f(noun_vec) if mode in (1, 2) else None, self.temperature, mode)
        mask = ops.positives_mask_from_tags(verb_vec, noun_vec, self._mode())           # G > 512: kernel-per-stage path
        x = engine.SimMatrixFn.apply(text_embeds, video_embeds, 1e-8)
        return engine.NceLossFn.apply(x, mask, self.temperature)

    def gathered(self, text_local, video_local, verb_local, noun_local, gather, rank, world):
        """Data-parallel entry: local rows in, loss out; the packed all-gather happens inside (engine.GatherEgoNceFn)."""
        G, Cc = text_local.shape[0] * world, text_local.shape[1]
        if ops.egonce_fused_supported(G, Cc) and video_local.shape[1] == Cc:
            return engine.GatherEgoNceFn.apply(text_local, video_local, verb_local, noun_local, self.temperature,
                                               self._mode(), gather, rank)
        return None


class MaxMarginRankingLoss(nn.Module):
    def __init__(self, margin=0.2, fix_norm=True):
        super().__init__()
        self.fix_norm, self.margin = fix_norm, margin

    def forward(self, x, weight=None):
        return engine.MaxMarginFn.apply(x, self.margin, self.fix_norm)       # `weight` ignored, as the reference (:63-90)


class AdaptiveMaxMarginRankingLoss(nn.Module):
    """model/loss.py:92-133: the margin of anchor i is `weight[i] * margin` (EPIC-MIR fine-tuning with relevancy)."""

    def __init__(self, margin=0.4, fix_norm=True):
        super().__init__()
        self.fix_norm, self.margin = fix_norm, margin

    def forward(self, x, weight=None):
        if weight is None:
            raise AttributeError("AdaptiveMaxMarginRankingLoss needs `weight` [n] (the reference calls weight.unsqueeze)")
        return engine.MaxMarginFn.apply(x, self.margin, self.fix_norm, weight)


class CrossEntropy(nn.Module):
    """model/loss.py:135-141: nn.CrossEntropyLoss() with its defaults (mean over the rows whose target is not -100, no
    class weights, no label smoothing) on the cross-entropy kernels.  The reference's callers
    (trainer/trainer_oscc.py:337, trainer/trainer_pnr.py:348) pass [G, C] logits and int64 class indices; other target
    forms (class probabilities, extra dimensions) are not implemented.  A class index outside [0, C) gives a NaN loss
    where torch raises a device assert."""

    ignore_index = -100

    def forward(self, output, target):
        if output.dim() != 2 or target.dim() != 1 or target.dtype != torch.int64 or target.shape[0] != output.shape[0]:
            raise NotImplementedError(f"CrossEntropy: [G, C] logits and int64 class indices [G] expected, got "
                                      f"{tuple(output.shape)} {output.dtype} and {tuple(target.shape)} {target.dtype}")
        return engine.CrossEntropyFn.apply(output, target.to(output.device), self.ignore_index)
