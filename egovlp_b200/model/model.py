"""FrozenInTime dual encoder + sim_matrix on the project's H100 kernels.

API mirror of the reference's model/model.py: FrozenInTime(video_params, text_params, projection_dim,
load_checkpoint, projection, load_temporal_fix), forward(data, video_only, return_embeds), compute_text,
compute_text_tokens, compute_video, set_device, sim_matrix(a, b, eps) -- and identical state_dict keys
(SURVEY.md section 8b), so reference checkpoints load and the unchanged trainer drives it.
"""
import os
import warnings

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import engine
from .video_transformer import SpaceTimeTransformer


def state_dict_data_parallel_fix(load_state_dict, curr_state_dict):
    """Strip / add the DataParallel 'module.' prefix so that `load` matches `curr` (reference utils/util.py:25-51)."""
    load_keys, curr_keys = list(load_state_dict.keys()), list(curr_state_dict.keys())
    if not load_keys or not curr_keys:
        return load_state_dict
    have, want = load_keys[0].startswith('module.'), curr_keys[0].startswith('module.')
    if have and not want:
        return type(load_state_dict)((k[len('module.'):], v) for k, v in load_state_dict.items())
    if want and not have:
        return type(load_state_dict)(('module.' + k, v) for k, v in load_state_dict.items())
    return load_state_dict


class BaseModel(nn.Module):
    """Reference base/base_model.py: __str__ appends the trainable-parameter count."""

    def __str__(self):
        n = sum(int(np.prod(p.size())) for p in self.parameters() if p.requires_grad)
        return super().__str__() + '\nTrainable parameters: {}'.format(n)


def _build_distilbert(text_params):
    """Parameter container for the text tower: HuggingFace DistilBertModel (weights only; its forward is not used).
    Loads the pretrained files when present, otherwise random-initialises the same architecture."""
    from transformers import DistilBertConfig, DistilBertModel
    cache_dir = 'pretrained/distilbert-base-uncased'
    try:
        from transformers import AutoModel
        return AutoModel.from_pretrained('distilbert-base-uncased', cache_dir=cache_dir, local_files_only=True)
    except Exception:  # no network / no files: synthetic-weights path
        warnings.warn("distilbert-base-uncased files not found: text tower is randomly initialised")
        return DistilBertModel(DistilBertConfig())


# Architectures a `bert*` name random-initialises to when its files are not present:
# (hidden_size, num_hidden_layers, num_attention_heads, intermediate_size, vocab_size)
_BERT_ARCHS = {'bert-base-uncased': (768, 12, 12, 3072, 30522), 'bert-base-cased': (768, 12, 12, 3072, 28996),
               'bert-large-uncased': (1024, 24, 16, 4096, 30522), 'bert-large-cased': (1024, 24, 16, 4096, 28996)}


def _build_bert(name):
    """Parameter container for a `bert*` text tower (reference model/model.py:34-35): the HuggingFace BertModel of
    `name` (weights only; its forward is not used).  Loads the local files when present, otherwise random-initialises
    the named architecture; any other name without files raises."""
    from transformers import AutoModel, BertConfig, BertModel
    try:
        return AutoModel.from_pretrained(name, local_files_only=True)
    except Exception:  # no network / no files: synthetic-weights path
        if name not in _BERT_ARCHS:
            raise NotImplementedError(f"{name}: no local files, and not one of {sorted(_BERT_ARCHS)} whose "
                                      "architecture can be random-initialised without them")
        warnings.warn(f"{name} files not found: text tower is randomly initialised")
        hid, layers, heads, inter, vocab = _BERT_ARCHS[name]
        return BertModel(BertConfig(hidden_size=hid, num_hidden_layers=layers, num_attention_heads=heads,
                                    intermediate_size=inter, vocab_size=vocab))


def _check_bert(tm):
    """Refuse, naming the field, a BERT the CUDA tower does not run: it takes the post-LN encoder with absolute
    positions, exact GELU, head dim 64, hidden <= 1024 and the pooler."""
    from transformers import BertModel
    if not isinstance(tm, BertModel):
        raise NotImplementedError(f"text model {type(tm).__name__}: only BertModel runs as a `bert*` text tower")
    cfg = tm.config
    if cfg.hidden_size % cfg.num_attention_heads or cfg.hidden_size // cfg.num_attention_heads != 64:
        raise NotImplementedError(f"num_attention_heads={cfg.num_attention_heads}: the text tower needs head dim 64 "
                                  f"(hidden_size={cfg.hidden_size})")
    if cfg.hidden_size > 1024:
        raise NotImplementedError(f"hidden_size={cfg.hidden_size}: the text tower takes hidden_size <= 1024")
    if cfg.hidden_act != 'gelu':
        raise NotImplementedError(f"hidden_act={cfg.hidden_act!r}: the text tower implements 'gelu' (exact erf)")
    if getattr(cfg, 'position_embedding_type', 'absolute') != 'absolute':
        raise NotImplementedError(f"position_embedding_type={cfg.position_embedding_type!r}: the text tower "
                                  "implements 'absolute'")
    if cfg.is_decoder or getattr(cfg, 'add_cross_attention', False):
        raise NotImplementedError("is_decoder / add_cross_attention: the text tower is an encoder")
    if tm.pooler is None:
        raise NotImplementedError("pooler: a BertModel built with add_pooling_layer=False has no pooler_output")


_VIT_B16_FILE = "pretrained/jx_vit_base_p16_224-80ecf9dd.pth"


def resample_pos_embed(pos_embed, grid):
    """A spatial positional embedding [1, 1 + n*n, D] of a square n x n patch grid, resampled to grid = (rows, cols):
    the patch part bicubically as a 2-D grid (F.interpolate, align_corners=False, computed in fp32), the CLS entry kept.
    Returned in pos_embed's dtype, on its device."""
    n = int(round((pos_embed.shape[1] - 1) ** 0.5))
    if pos_embed.dim() != 3 or pos_embed.shape[0] != 1 or n * n != pos_embed.shape[1] - 1:
        raise NotImplementedError(f"pos_embed of shape {tuple(pos_embed.shape)}: only a square patch grid can be "
                                  "resampled")
    D = pos_embed.shape[2]
    patch = pos_embed[:, 1:].float().reshape(1, n, n, D).permute(0, 3, 1, 2)
    patch = F.interpolate(patch, size=tuple(grid), mode="bicubic", align_corners=False)
    patch = patch.permute(0, 2, 3, 1).reshape(1, grid[0] * grid[1], D)
    return torch.cat([pos_embed[:, :1].float(), patch], 1).to(pos_embed.dtype)


def _build_video_tower(video_params, from_scratch):
    """SpaceTimeTransformer exactly as the reference configures it (model/model.py:43-66): defaults for missing keys,
    ImageNet ViT-B/16 weights for a tower that is not restored from a checkpoint, identity head / pre_logits / fc."""
    kind = video_params['model']
    if kind != "SpaceTimeTransformer":
        raise NotImplementedError(f"{kind} not implemented")
    opts = {'num_frames': 4, 'time_init': 'zeros', 'attention_style': 'frozen-in-time', 'arch_config': 'base_patch16_224'}
    opts.update({k: video_params[k] for k in opts if k in video_params})
    if opts.pop('arch_config') != 'base_patch16_224':
        raise NotImplementedError
    # frame size (another key the reference does not read); pretrained pos_embed grids are resampled to it on load
    img_size = video_params.get('img_size', 224)
    if isinstance(img_size, bool) or not isinstance(img_size, int) or img_size < 16:
        raise ValueError(f"video_params['img_size'] must be an int >= 16, got {img_size!r}")
    tower = SpaceTimeTransformer(img_size=img_size, **opts)
    tower.head = tower.pre_logits = tower.fc = nn.Identity()      # `fc`: "backwards compatibility (old models)"
    # selective activation recompute in training (a key the reference does not read: its configs load unchanged there)
    tower.set_grad_checkpointing(bool(video_params.get('grad_checkpointing', False)))
    # e4m3 inference GEMMs, opt-in (another key the reference does not read)
    tower.set_inference_precision(video_params.get('inference_precision', 'bf16'))
    if from_scratch:
        if os.path.exists(_VIT_B16_FILE):
            vit = state_dict_data_parallel_fix(torch.load(_VIT_B16_FILE, map_location="cpu"), tower.state_dict())
            if 'img_size' in video_params and 'pos_embed' in vit:
                vit['pos_embed'] = resample_pos_embed(vit['pos_embed'], tower.pos_embed_grid())
            tower.load_state_dict(vit, strict=False)
        else:
            warnings.warn(f"{_VIT_B16_FILE} not found: video tower keeps its random initialisation")
    return tower


class FrozenInTime(BaseModel):
    def __init__(self, video_params, text_params, projection_dim=256, load_checkpoint=None, projection='minimal',
                 load_temporal_fix='zeros'):
        super().__init__()
        self.video_params, self.text_params, self.load_temporal_fix = video_params, text_params, load_temporal_fix
        if not text_params['pretrained']:
            raise NotImplementedError("Huggingface text models require pretrained init.")
        name = text_params['model']
        self._bert = name.startswith('bert')
        if self._bert:
            self.text_model = _build_bert(name)
            _check_bert(self.text_model)
        elif name.startswith('distilbert'):
            self.text_model = _build_distilbert(text_params)
        else:
            raise NotImplementedError(f"{name}: the text tower implements DistilBERT (`distilbert*`) and BERT "
                                      "(`bert*`)")
        self.text_model.train()                                   # as the reference: HF dropouts active while training
        restoring = load_checkpoint not in ("", None)
        self.video_model = _build_video_tower(video_params, from_scratch=not restoring)

        if projection == 'minimal':                               # project both towers to the common embedding
            self.txt_proj = nn.Sequential(nn.ReLU(), nn.Linear(self.text_model.config.hidden_size, projection_dim))
            self.vid_proj = nn.Sequential(nn.Linear(self.video_model.embed_dim, projection_dim))
        elif projection == '':
            self.txt_proj, self.vid_proj = nn.Identity(), nn.Identity()
        else:
            raise NotImplementedError
        object.__setattr__(self, "_bf16_cache", self.video_model._bf16_cache)
        if restoring:
            self._restore(load_checkpoint)

    def _restore(self, path):
        """model/model.py:88-95: a trainer checkpoint, saved with or without the DataParallel prefix and possibly with
        a different number of frames."""
        rank = int(os.environ.get('LOCAL_RANK', 0))
        where = f'cuda:{rank}' if torch.cuda.is_available() else 'cpu'
        saved = torch.load(path, map_location=where, weights_only=False)['state_dict']
        saved = self._inflate_positional_embeds(state_dict_data_parallel_fix(saved, self.state_dict()))
        self.load_state_dict(saved, strict=True)

    def set_device(self, device):
        self.device = device

    def forward(self, data, video_only=False, return_embeds=True):
        if video_only:
            return self.compute_video(data['video'])
        if torch.is_grad_enabled():
            self._bf16_cache.refresh()           # once per training forward (both towers share the cache)
        text_embeddings = self._text(data['text'], False, _refresh=False)
        video_embeddings = self.compute_video(data['video'], _refresh=False)
        if return_embeds:
            return text_embeddings, video_embeddings
        return sim_matrix(text_embeddings, video_embeddings)

    # ---- text ------------------------------------------------------------------------------------------------
    def _text_params(self):
        tm = self.text_model
        if self._bert:
            e = tm.embeddings
            p = [e.word_embeddings.weight, e.position_embeddings.weight, e.token_type_embeddings.weight,
                 e.LayerNorm.weight, e.LayerNorm.bias]
            for layer in tm.encoder.layer:
                a = layer.attention
                for lin in (a.self.query, a.self.key, a.self.value, a.output.dense):
                    p += [lin.weight, lin.bias]
                p += [a.output.LayerNorm.weight, a.output.LayerNorm.bias, layer.intermediate.dense.weight,
                      layer.intermediate.dense.bias, layer.output.dense.weight, layer.output.dense.bias,
                      layer.output.LayerNorm.weight, layer.output.LayerNorm.bias]
            return p + [tm.pooler.dense.weight, tm.pooler.dense.bias]
        p = [tm.embeddings.word_embeddings.weight, tm.embeddings.position_embeddings.weight,
             tm.embeddings.LayerNorm.weight, tm.embeddings.LayerNorm.bias]
        for layer in tm.transformer.layer:
            a, f = layer.attention, layer.ffn
            for lin in (a.q_lin, a.k_lin, a.v_lin, a.out_lin):
                p += [lin.weight, lin.bias]
            p += [layer.sa_layer_norm.weight, layer.sa_layer_norm.bias, f.lin1.weight, f.lin1.bias, f.lin2.weight,
                  f.lin2.bias, layer.output_layer_norm.weight, layer.output_layer_norm.bias]
        return p

    def _text(self, text_data, tokens_mode, _refresh=True):
        # projection='' (nn.Identity, reference :80-82): the tower ends at the DistilBERT hidden state / the BERT pooler
        # output (no ReLU / Linear)
        proj = self.txt_proj[1] if isinstance(self.txt_proj, nn.Sequential) else None
        cfg = self.text_model.config
        if _refresh and torch.is_grad_enabled():
            self._bf16_cache.refresh()
        # train-mode dropouts of the HF text model (the reference keeps `text_model.train()`, :36); eval() or a config
        # with dropout = attention_dropout = 0 gives the deterministic path
        # (BERT: input_ids and attention_mask only -- the reference passes no token_type_ids, so every token gets
        # token type 0, and its compute_text_tokens returns the pooled output as compute_text does, :129-131)
        if self._bert:
            drop = ((cfg.hidden_dropout_prob, cfg.attention_probs_dropout_prob) if self.text_model.training
                    else (0.0, 0.0))
            return engine.BertTowerFn.apply(text_data['input_ids'], text_data['attention_mask'],
                                            cfg.num_attention_heads, cfg.layer_norm_eps,
                                            (False, torch.is_grad_enabled()), self._bf16_cache, drop,
                                            *self._text_params(),
                                            *((proj.weight, proj.bias) if proj is not None else (None, None)))
        drop = (cfg.dropout, cfg.attention_dropout) if self.text_model.training else (0.0, 0.0)
        return engine.TextTowerFn.apply(text_data['input_ids'], text_data['attention_mask'], cfg.n_heads, 1e-12,
                                        (tokens_mode, torch.is_grad_enabled()), self._bf16_cache, drop, *self._text_params(),
                                        *((proj.weight, proj.bias) if proj is not None else (None, None)))

    def compute_text(self, text_data):
        return self._text(text_data, False)

    def compute_text_tokens(self, text_data):
        return self._text(text_data, True)

    # ---- video -----------------------------------------------------------------------------------------------
    def compute_video(self, video_data, _refresh=True):
        proj = self.vid_proj[0] if isinstance(self.vid_proj, nn.Sequential) else None
        return self.video_model.forward_features(video_data, proj=proj, _refresh=_refresh)

    # ---- checkpoint compat -----------------------------------------------------------------------------------
    def _inflate_positional_embeds(self, new_state_dict):
        """Load a checkpoint trained with a different number of frames (reference :145-187): truncate, or extend
        with zeros / nearest / bilinear interpolation along the frame axis.  A pos_embed of another patch grid is
        resampled to the tower's (resample_pos_embed) when video_params sets 'img_size'; without that key it is
        refused, as the reference refuses it."""
        key = 'video_model.temporal_embed'
        curr = self.state_dict()
        if key in new_state_dict and key in curr:
            load_te = new_state_dict[key]
            load_f, curr_f = load_te.shape[1], self.video_params['num_frames']
            if load_f > curr_f:
                new_state_dict[key] = load_te[:, :curr_f, :]
            elif load_f < curr_f:
                if self.load_temporal_fix == 'zeros':
                    new_te = torch.zeros([load_te.shape[0], curr_f, load_te.shape[2]], dtype=load_te.dtype,
                                         device=load_te.device)
                    new_te[:, :load_f] = load_te
                elif self.load_temporal_fix in ['interp', 'bilinear']:
                    mode = 'bilinear' if self.load_temporal_fix == 'bilinear' else 'nearest'
                    kw = dict(align_corners=True) if mode == 'bilinear' else {}
                    new_te = F.interpolate(load_te.unsqueeze(0), (curr_f, load_te.shape[2]), mode=mode, **kw).squeeze(0)
                else:
                    raise NotImplementedError
                new_state_dict[key] = new_te
        key = 'video_model.pos_embed'
        if key in new_state_dict and key in curr and new_state_dict[key].shape[1] != curr[key].shape[1]:
            if 'img_size' not in self.video_params:
                raise NotImplementedError(
                    'Loading models with different spatial resolution / patch number not yet implemented, sorry.')
            new_state_dict[key] = resample_pos_embed(new_state_dict[key], self.video_model.pos_embed_grid())
        return new_state_dict


def sim_matrix(a, b, eps=1e-8):
    """Cosine similarity a_n @ b_n^T with norms clamped at eps (reference model/model.py:189-197).  Host tensors (the
    reference's evaluation loops move embeddings to the host first) are computed on the current CUDA device and the
    result comes back to the host; the copies are ordinary `.to()` calls, so autograd sees them.  Without CUDA this
    raises, like every other op of the package."""
    if a.device != b.device:
        raise RuntimeError(f"sim_matrix: expected both inputs on the same device, got {a.device} and {b.device}")
    if a.device.type == "cpu" and torch.cuda.is_available():
        dev = torch.device("cuda", torch.cuda.current_device())
        return engine.SimMatrixFn.apply(a.to(dev), b.to(dev), eps).to(a.device)
    return engine.SimMatrixFn.apply(a, b, eps)
