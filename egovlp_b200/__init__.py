"""egovlp_b200: H100-native (sm_90a) implementation of the EgoVLP dual-encoder pretraining hot path.

    from egovlp_b200.model.model import FrozenInTime, sim_matrix
    from egovlp_b200.model.loss import EgoNCE, NormSoftmaxLoss, MaxMarginRankingLoss

`install_as_reference_model()` aliases the package under the reference's module names (`model.model`,
`model.loss`, `model.video_transformer`, `model.metric`) so the reference's run/ and trainer/ scripts import it
unchanged (see INTEGRATION.md).
"""
import importlib
import sys

__version__ = "0.1.0"


def _one_bucket_ddp():
    """Make `DistributedDataParallel(...)` calls that do not choose a bucket size (the reference's
    base/base_trainer.py:254-258) use ONE gradient bucket all-reduced after the backward: with this package's persistent
    one-CTA-per-SM GEMMs, NCCL's CTAs competing with the persistent GEMMs of the backward cost more than overlapped
    25 MB buckets hide (measured on an earlier multi-GPU Blackwell build; not re-measured on H100).
    EGOVLP_DDP_BUCKET_MB overrides (25 = torch's default)."""
    import functools
    import os
    import torch
    ddp = torch.nn.parallel.DistributedDataParallel
    if getattr(ddp.__init__, "_egovlp_bucket_default", False):
        return
    orig = ddp.__init__

    @functools.wraps(orig)
    def init(self, *args, **kwargs):
        kwargs.setdefault("bucket_cap_mb", int(os.environ.get("EGOVLP_DDP_BUCKET_MB", "2048")))
        orig(self, *args, **kwargs)

    init._egovlp_bucket_default = True
    ddp.__init__ = init


def install_as_reference_model(patch_optimizer=True, one_bucket_ddp=True):
    """Alias the package under the reference's module names.  With `patch_optimizer` the optimizer the reference's
    configs name -- `getattr(transformers, 'AdamW')`, run/train_egoclip.py:72-73 -- resolves to the fused
    egovlp_b200.optim.AdamW (same HF semantics; transformers 5.x removed the class).  Any other optimizer keeps
    working: the bf16 weight copies are refreshed every training forward (engine.Bf16Cache.refresh).  With
    `one_bucket_ddp` the trainer's DistributedDataParallel wrapper all-reduces one gradient bucket after the backward."""
    pkg = importlib.import_module("egovlp_b200.model")
    sys.modules["model"] = pkg
    for name in ("model", "loss", "video_transformer", "metric"):
        sys.modules["model." + name] = importlib.import_module("egovlp_b200.model." + name)
    if patch_optimizer:
        import transformers
        from .optim import AdamW
        transformers.AdamW = AdamW
    if one_bucket_ddp:
        _one_bucket_ddp()
    return pkg
