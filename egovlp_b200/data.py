"""Input feed helpers (SURVEY.md section 8f row 2): the reference trainer moves every batch with blocking fp32
`.to(device)` calls (trainer/trainer_egoclip.py:118-121, 616 MB/step at 64 x 16 frames).  `DevicePrefetcher`
keeps one batch in flight on a side stream from pinned host memory; frames may stay uint8 (4x fewer bytes) because
the patch-embedding kernel normalises them on the GPU."""
import torch


def _to_device(obj, device):
    if torch.is_tensor(obj):
        return obj.to(device, non_blocking=True)
    if isinstance(obj, dict):
        return {k: _to_device(v, device) for k, v in obj.items()}
    if isinstance(obj, (list, tuple)):
        return type(obj)(_to_device(v, device) for v in obj)
    return obj


def _record(obj, stream):
    if torch.is_tensor(obj):
        obj.record_stream(stream)
    elif isinstance(obj, dict):
        for v in obj.values():
            _record(v, stream)
    elif isinstance(obj, (list, tuple)):
        for v in obj:
            _record(v, stream)


class DevicePrefetcher:
    """Iterates `loader` (batches of pinned host tensors / nested dicts) one batch ahead on a copy stream.
    `transform`, if given, is called on each batch on the copy stream after its H2D copy (e.g.
    `transforms.DeviceVideoTransform`, which turns packed uint8 clips into the model's fp32 frames)."""

    def __init__(self, loader, device, transform=None):
        self.loader, self.device, self.transform = loader, torch.device(device), transform
        self.stream = torch.cuda.Stream(device=self.device)

    def __iter__(self):
        it = iter(self.loader)
        nxt = self._fetch(it)
        while nxt is not None:
            torch.cuda.current_stream(self.device).wait_stream(self.stream)
            cur = nxt
            _record(cur, torch.cuda.current_stream(self.device))
            nxt = self._fetch(it)
            yield cur

    def _fetch(self, it):
        try:
            batch = next(it)
        except StopIteration:
            return None
        with torch.cuda.stream(self.stream):
            batch = _to_device(batch, self.device)
            return batch if self.transform is None else self.transform(batch)
