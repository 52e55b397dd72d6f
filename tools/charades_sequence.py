"""The reference's Charades-Ego trainer, call for call (trainer/trainer_charades.py): the training step (:104-145), the
learning-rate schedule (:77-82) and the zero-shot / fine-tuned evaluation `_valid_epoch` (:167-250), driving the package
through the reference-facing API only: `model(data)`, `sim_matrix`, `NormSoftmaxLoss`, an HF-style optimizer and the
metric functions the config names.

Test / benchmark infrastructure (tests/test_charades_gpu.py, tools/bench_charades.py), like tools/trainer_sequence.py:
the real trainer file is unchanged, and this restatement lets the sequence it runs -- including the host-side `cat` of
the embeddings, `sim_matrix` on host tensors and `.numpy().T` -- be checked and measured where the reference does not
exist."""
import torch
import torch.distributed as dist

from tools.trainer_sequence import AllGatherMulti, dist_args


def adjust_learning_rate(optimizer, epoch, args):
    """trainer_charades.py:77-82: lr = learning_rate1, times 0.1 for every milestone of `schedule` already reached."""
    lr = args.learning_rate1
    for milestone in args.schedule:
        lr *= 0.1 if epoch >= milestone else 1.
    for param_group in optimizer.param_groups:
        param_group['lr'] = lr


def train_step(model, loss_fn, optimizer, host_batch, device, sim_matrix, args=None, n_gpu=1):
    """One iteration of the loop body at trainer_charades.py:109-145 on an already tokenised host batch
    {'video', 'text': {'input_ids', 'attention_mask'}}.  Returns `loss.detach().item()` (:135)."""
    args = args or dist_args()
    data = dict(host_batch)
    data['text'] = {key: val.to(device) for key, val in data['text'].items()}            # :114
    data['video'] = data['video'].to(device)                                             # :115
    optimizer.zero_grad()                                                                # :117
    with torch.set_grad_enabled(True):
        text_embeds, video_embeds = model(data)                                          # :119
        video_embeds = AllGatherMulti.apply(video_embeds, n_gpu, args)                   # :120
        text_embeds = AllGatherMulti.apply(text_embeds, n_gpu, args)                     # :121
        output = sim_matrix(text_embeds, video_embeds)                                   # :122
        loss = loss_fn(output)                                                           # :123
    loss.backward()                                                                      # :124
    optimizer.step()                                                                     # :126
    total = loss.detach().item()                                                         # :135
    optimizer.zero_grad()                                                                # :145
    return total


def _gather(t):
    """trainer_charades.py:212-214 / :217-219: list-API all_gather + cat (identity at world size 1)."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return t
    out = [torch.zeros_like(t) for _ in range(dist.get_world_size())]
    dist.all_gather(out, t)
    return torch.cat(out, dim=0)


def valid_epoch(model, prompts, host_batches, device, sim_matrix, metrics, dummy_video=None):
    """trainer_charades.py:176-243 for one validation loader.  `prompts` = the tokenised class prompts (:194),
    `host_batches` = [{'video', 'text', 'target'}, ...] host tensors, `metrics` = the config's metric functions.
    The dummy video of the class-prompt forward (:197, uninitialised `torch.Tensor(1, 4, 3, 224, 224)` unless given)
    goes to the device, as the DistributedDataParallel / DataParallel wrapper moves its inputs.
    -> ({metric name: result}, sims [videos, classes] numpy, text_embeds, vid_embeds (host tensors))."""
    model.eval()                                                                         # :176
    with torch.no_grad():
        data_cls = {key: val.to(device) for key, val in prompts.items()}                 # :195
        video = torch.Tensor(1, 4, 3, 224, 224) if dummy_video is None else dummy_video
        dict_cls = {'text': data_cls, 'video': video.to(device)}                         # :197
        text_embed, _ = model(dict_cls, return_embeds=True)                              # :198
        text_embeds = text_embed.cpu().detach()                                          # :199
        vid_embed_arr, target_arr = [], []
        for host in host_batches:
            data = dict(host)
            data['text'] = {key: val.to(device) for key, val in data['text'].items()}    # :206
            data['video'] = data['video'].to(device)                                     # :207
            data_target = data['target'].to(device)                                      # :208
            _, vid_embed = model(data, return_embeds=True)                               # :210
            vid_embed_arr.append(_gather(vid_embed).cpu())                               # :212-215
            target_arr.append(_gather(data_target).cpu())                                # :217-220
    vid_embeds = torch.cat(vid_embed_arr)                                                # :235
    target_embeds = torch.cat(target_arr)                                                # :236
    sims = sim_matrix(text_embeds, vid_embeds).numpy().T                                 # :238
    targets = target_embeds.numpy()                                                      # :239
    res = {metric.__name__: metric(sims, targets) for metric in metrics}                 # :241-243
    return res, sims, text_embeds, vid_embeds
