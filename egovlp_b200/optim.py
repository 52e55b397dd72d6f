"""AdamW with HuggingFace `transformers.AdamW` semantics (the optimizer type the reference's configs name;
removed from transformers 5.x) on one fused multi-tensor CUDA kernel."""
import ctypes as C
import math

import torch

from ._lib import call, lib


class _TensorDesc(C.Structure):
    _fields_ = [("param", C.c_void_p), ("grad", C.c_void_p), ("exp_avg", C.c_void_p), ("exp_avg_sq", C.c_void_p),
                ("numel", C.c_longlong), ("shadow_bf16", C.c_void_p)]


class AdamW(torch.optim.Optimizer):
    """transformers.AdamW(params, lr=1e-3, betas=(0.9, 0.999), eps=1e-6, weight_decay=0.0, correct_bias=True).

    One kernel launch per (param group, step count): HF keeps a step counter PER PARAMETER, so parameters that started
    receiving gradients later (unfrozen mid-run, partial optimizer-state load) get their own bias correction -- they are
    launched as a separate sub-group instead of sharing the first parameter's count.  The bf16 GEMM-operand copies
    that `engine.Bf16Cache` holds for a parameter are rewritten in the same pass (`shadow_bf16`): a forward that reads
    them without `Bf16Cache.refresh()` -- an evaluation right after a step -- finds them current and casts nothing.  A
    training forward re-casts every copy in `refresh()` regardless, since a write through `p.data` after the step would
    not show in `p._version`."""

    _egovlp_fused = True          # engine's optimizer-step hook: this optimizer keeps the bf16 copies current itself
    _RING = 4                     # pinned staging buffers for the descriptor table (pointers move with zero_grad)

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-6, weight_decay=0.0, correct_bias=True):
        if lr < 0.0 or not 0.0 <= betas[0] < 1.0 or not 0.0 <= betas[1] < 1.0 or eps < 0.0:
            raise ValueError("invalid AdamW hyper-parameters")
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, correct_bias=correct_bias))
        self._tables = {}

    def _table(self, slot, plist, shadows):
        """Device-side descriptor table of one launch.  The chunk map depends only on the tensor sizes and is built
        once; the pointer table is re-staged (pinned host ring -> async copy on the launch stream) whenever a tensor
        moved -- typically the .grad pointers after zero_grad(set_to_none=True) -- never from pageable memory."""
        key = tuple((p.data_ptr(), p.grad.data_ptr(), self.state[p]["exp_avg"].data_ptr(),
                     self.state[p]["exp_avg_sq"].data_ptr(), sh.t16.data_ptr() if sh is not None else 0)
                    for p, sh in zip(plist, shadows))
        sizes = tuple(p.numel() for p in plist)
        ent = self._tables.get(slot)
        dev = plist[0].device
        if ent is None or ent["sizes"] != sizes or ent["dev"].device != dev:
            chunk = lib().egovlp_adamw_chunk_elems()
            ct, co = [], []
            for i, n_el in enumerate(sizes):
                n = (n_el + chunk - 1) // chunk
                ct += [i] * n
                co += list(range(n))
            nbytes = C.sizeof(_TensorDesc) * len(plist)
            ent = {"sizes": sizes, "key": None, "turn": 0,
                   "dev": torch.empty(nbytes, dtype=torch.uint8, device=dev),
                   "ring": [torch.empty(nbytes, dtype=torch.uint8).pin_memory() for _ in range(self._RING)],
                   "events": [None] * self._RING,
                   "ct": torch.tensor(ct, dtype=torch.int32, device=dev),
                   "co": torch.tensor(co, dtype=torch.int32, device=dev)}
            self._tables[slot] = ent
        if ent["key"] != key:
            descs = (_TensorDesc * len(plist))()
            for i, (k, p) in enumerate(zip(key, plist)):
                descs[i] = _TensorDesc(k[0], k[1], k[2], k[3], p.numel(), k[4] or None)
            turn = ent["turn"]
            if ent["events"][turn] is not None:
                ent["events"][turn].synchronize()             # the copy that last used this staging buffer is done
            host = ent["ring"][turn]
            C.memmove(host.data_ptr(), C.addressof(descs), C.sizeof(descs))
            ent["dev"].copy_(host, non_blocking=True)
            ev = torch.cuda.Event()
            ev.record()
            ent["events"][turn] = ev
            ent["turn"] = (turn + 1) % self._RING
            ent["key"] = key
        return ent["dev"], ent["ct"], ent["co"]

    @torch.no_grad()
    def step(self, closure=None):
        from . import engine
        loss = closure() if closure is not None else None
        for gi, group in enumerate(self.param_groups):
            by_step = {}
            for p in group["params"]:
                if p.grad is None:
                    continue
                st = self.state[p]
                if not st:
                    st["step"] = 0
                    st["exp_avg"] = torch.zeros_like(p, memory_format=torch.contiguous_format)
                    st["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.contiguous_format)
                assert p.is_cuda and p.dtype == torch.float32 and p.is_contiguous() and p.grad.is_contiguous()
                assert p.grad.dtype == torch.float32, "AdamW: fp32 gradients expected"
                st["step"] = int(st["step"]) + 1
                by_step.setdefault(st["step"], []).append(p)
            b1, b2 = group["betas"]
            for si, (t, plist) in enumerate(sorted(by_step.items())):
                step_size = group["lr"]
                if group["correct_bias"]:
                    step_size = step_size * math.sqrt(1.0 - b2 ** t) / (1.0 - b1 ** t)
                shadows = []
                for p in plist:
                    sh = engine.shadow_entry(p)
                    shadows.append(sh if sh is not None and sh.t16.is_contiguous() and sh.t16.numel() == p.numel() else None)
                with torch.cuda.device(plist[0].device):
                    raw, ct, co = self._table((gi, si), plist, shadows)
                    call("egovlp_adamw_multi", C.c_void_p(raw.data_ptr()), C.c_void_p(ct.data_ptr()),
                         C.c_void_p(co.data_ptr()), ct.numel(), C.c_float(group["lr"]), C.c_float(b1), C.c_float(b2),
                         C.c_float(group["eps"]), C.c_float(group["weight_decay"]), C.c_float(step_size), C.c_void_p(0),
                         C.c_void_p(torch.cuda.current_stream().cuda_stream))
                for p, sh in zip(plist, shadows):
                    torch.autograd.graph.increment_version(p)   # the kernel wrote p.data: autograd / caches must see it
                    if sh is not None:
                        sh.stamp(p)                             # ... and its bf16 copy is current for Bf16Cache.get()
        return loss
