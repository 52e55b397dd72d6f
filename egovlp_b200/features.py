"""Dense feature extraction with the dual encoder (SURVEY.md 8f row 4): the loops of the reference's
run/test_nlq.py:60-109 (also run/test_mq.py) as library functions.  The reference pushes windows through
`model.compute_video` four at a time (`batch = 4`, :78); per-window results do not depend on the batch (every kernel
on the forward path is row-independent and the forward GEMMs use no split-K), so a large batch gives
bit-identical features."""
import torch


@torch.no_grad()
def dense_video_features(model, frames, num_frames, batch=64, reference_tail=False):
    """frames [F, 3, H, W] (one whole clip, fp32 normalised) -> [F // num_frames, projection_dim] on the CPU, one
    feature per consecutive `num_frames`-frame window (run/test_nlq.py:69-86).

    reference_tail=True reproduces the reference loop exactly: it runs `windows // batch` full batches and leaves
    the features of the trailing `windows % batch` windows at zero (:79-86)."""
    f = frames.shape[0]
    windows = frames[: f // num_frames * num_frames].reshape(-1, num_frames, *frames.shape[1:])
    n = windows.shape[0]
    dim = model.vid_proj[0].out_features if isinstance(model.vid_proj, torch.nn.Sequential) else model.video_model.embed_dim
    outs = torch.zeros(n, dim)
    stop = n // batch * batch if reference_tail else n
    for start in range(0, stop, batch):
        chunk = windows[start:min(start + batch, stop)].to(model.device, non_blocking=True)
        outs[start:start + chunk.shape[0]] = model.compute_video(chunk).float().cpu()
    return outs


@torch.no_grad()
def text_features(model, text, token=False):
    """text = tokenizer output on `model.device` (dict of input_ids / attention_mask).  token=False: the sentence
    embedding `compute_text` [B, C].  token=True: per-word embeddings of the FIRST sample without [CLS] / [SEP]
    (run/test_nlq.py:99-102): `compute_text_tokens(text)[0][1 : num_words - 1]`."""
    if not token:
        return model.compute_text(text)
    emb = model.compute_text_tokens(text)[0]
    num_words = int(text["attention_mask"][0].sum())
    return emb[1:num_words - 1]
