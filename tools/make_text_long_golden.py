"""Generate tests/golden/distilbert_long.npz: HF DistilBertModel (the installed transformers, eval mode) on captions
up to its 512 positions, the recording tests/test_text_long_gpu.py checks the oracle and the text tower against.

    python tools/make_text_long_golden.py

Config: dim 128, 2 heads (head dim 64), 2 layers, hidden 256, vocab 120, max_position_embeddings 512; weights are
egovlp_b200.synthetic.seeded_state_dict(LONG_DIMS, seed=SEED).  Inputs: L = 512 with valid lengths 512, 300, 129,
65, 7 and one non-prefix mask (holes inside the valid range); a second call at L = 200 on the same captions cut to
200.  Stored: every hidden state's CLS rows plus 64 seeded token rows per call (the whole tensors are ~5 MB; the
fixture stays near 200 KB).
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from egovlp_b200 import synthetic as syn  # noqa: E402

LONG_DIMS = dict(syn.TINY_DIMS, max_pos=512)
SEED = 6
LENGTHS = (512, 300, 129, 65, 7)
SAMPLE_ROWS = 64


def inputs():
    """ids [6, 512] (CLS = 101 first, SEP = 102 last valid, 0 on padding) and masks: LENGTHS, then a holed row."""
    g = torch.Generator().manual_seed(17)
    B, L = len(LENGTHS) + 1, 512
    ids = torch.randint(103, 120, (B, L), generator=g)
    mask = torch.zeros(B, L, dtype=torch.int64)
    for b, n in enumerate(LENGTHS):
        mask[b, :n] = 1
    holed = torch.ones(L, dtype=torch.int64)
    holed[400:] = 0
    holed[30:70] = 0          # a whole 64-key tile's worth of holes across a tile edge
    holed[130:131] = 0
    holed[200:260:3] = 0
    mask[-1] = holed
    for b in range(B):
        last = int(mask[b].nonzero().max())
        ids[b, 0], ids[b, last] = 101, 102
    ids[mask == 0] = 0
    return ids, mask


def row_sample(B, L, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, B, (SAMPLE_ROWS,), generator=g), torch.randint(0, L, (SAMPLE_ROWS,), generator=g)


def main():
    from transformers import DistilBertConfig, DistilBertModel
    d = LONG_DIMS
    sd = syn.seeded_state_dict(d, seed=SEED, video=False, proj=False)
    cfg = DistilBertConfig(vocab_size=d["vocab"], dim=d["text_dim"], n_layers=d["text_layers"], n_heads=d["text_heads"],
                           hidden_dim=d["text_hidden"], max_position_embeddings=d["max_pos"], dropout=0.0,
                           attention_dropout=0.0)
    net = DistilBertModel(cfg).eval()
    print("load:", net.load_state_dict({k[len("text_model."):]: v for k, v in sd.items()}, strict=True))
    ids, mask = inputs()
    out = {"input_ids": ids.numpy(), "attention_mask": mask.numpy(), "seed": SEED}
    with torch.no_grad():
        for L, tag in ((512, "l512"), (200, "l200")):
            hs = torch.stack(net(input_ids=ids[:, :L], attention_mask=mask[:, :L], output_hidden_states=True).hidden_states)
            bi, li = row_sample(ids.shape[0], L, seed=L)
            out[f"{tag}_cls"] = hs[:, :, 0].numpy()                      # [layers + 1, B, D]
            out[f"{tag}_rows_b"], out[f"{tag}_rows_l"] = bi.numpy(), li.numpy()
            out[f"{tag}_rows"] = hs[:, bi, li].numpy()                   # [layers + 1, SAMPLE_ROWS, D]
    path = os.path.join(ROOT, "tests", "golden", "distilbert_long.npz")
    np.savez_compressed(path, **out)
    print(f"wrote {path}  ({os.path.getsize(path) / 1024:.1f} KiB)")


if __name__ == "__main__":
    main()
