"""CPU restatement (torch, functional) of the Ego4D OSCC / PNR fine-tuning pieces of the reference.  TEST
INFRASTRUCTURE ONLY, like oracle/reference_port.py (whose towers it builds on): imported by tests/ and
tools/bench_finetune.py's eager baseline, never by the product package.  Pinned against the unmodified reference by
oracle/make_finetune_golden.py -> tests/golden/finetune.npz (tests/test_finetune_oracle.py).  Every function names the
reference lines it restates."""
import torch


def cross_entropy(x, target, ignore_index=-100):
    """CrossEntropy.forward (model/loss.py:135-141) = nn.CrossEntropyLoss() with its defaults, written out: mean over
    the rows whose target is not ignore_index of logsumexp(x_r) - x_r[target_r]; no valid row gives 0 / 0 = NaN.  A
    target outside [0, C) that is not ignore_index gives NaN (torch raises instead)."""
    keep = target != ignore_index
    if bool(((target < 0) | (target >= x.shape[1]))[keep].any()):
        return torch.full((), float("nan"), dtype=x.dtype, device=x.device)
    t = torch.where(keep, target, torch.zeros_like(target))
    rows = torch.logsumexp(x, dim=1) - x.gather(1, t[:, None])[:, 0]
    return torch.where(keep, rows, torch.zeros_like(rows)).sum() / keep.sum()


def oscc_step_loss(scores_local, state_local):
    """trainer/trainer_oscc.py:334-337 for a list of per-rank local tensors: AllGather_multi (== cat) of the [B, 2]
    video-only scores and of the state labels, then CrossEntropy."""
    return cross_entropy(torch.cat(scores_local), torch.cat(state_local))


def pnr_step_loss(scores_local, labels_local, state_local):
    """trainer/trainer_pnr.py:341-348: torch.mean(state.T * CE(scores.squeeze(-1), argmax(labels.long(), 1))).  CE is
    already the scalar mean, so this is mean(state) * CE; clips without a state change still enter the CE."""
    scores, labels, state = torch.cat(scores_local), torch.cat(labels_local), torch.cat(state_local)
    return torch.mean(state.T * cross_entropy(scores.squeeze(dim=-1), torch.argmax(labels.long(), dim=1)))


def oscc_metrics(preds, labels):
    """model/metric.py:342-353: accuracy in % of the per-row argmax (ties -> lowest index)."""
    correct = sum(int(torch.argmax(p).item() == l.item()) for p, l in zip(preds, labels))
    return {"accuracy": correct / len(preds) * 100}


def pnr_metrics(preds, labels, sc_labels, fps, parent_start_frames, parent_end_frames, parent_pnr_frames):
    """model/metric.py:355-397: over the rows with sc_label == 1, |(end - start) / 16 * argmax - (pnr - start)| / fps
    with the mapped keyframe a TENSOR true division (float32 for integer frames) and the rest in Python floats; the
    mean of an empty list (NaN) when no row has a state change (:388-393 is overwritten by :394)."""
    import warnings
    import numpy as np
    errs = []
    for pred, sc, s, e, p, f in zip(preds, sc_labels, parent_start_frames, parent_end_frames, parent_pnr_frames, fps):
        if sc.item() == 1:
            mapped = ((e - s) / 16 * torch.argmax(pred).item()).item()
            errs.append(abs(mapped - (p.item() - s.item())) / f.item())
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)
        return {"keyframe_distance": np.mean(errs)}
