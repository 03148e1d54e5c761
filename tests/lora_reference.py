"""LoRA reference for the tests: the CPU oracle's LLaMA forward (oracle/macaw_oracle.py) with every adapted projection
computed as PEFT's LoRA linear (peft/tuners/lora/layer.py Linear.forward):

    y = x W^T + s * (drop(x) A^T) B^T,   drop(x) = x * mult

`mult` holds the explicit dropout multipliers (0 or 1/(1-p)) of one adapter, passed in the way the oracle's mha_forward
takes the attention-dropout ones, so the reference and the device use the SAME mask.  Without multipliers the formula is
PEFT's eval-mode forward.  The oracle itself is run unchanged: each adapted weight of its state dict is replaced by a
`LoraLinear`, which the oracle's `F.linear` calls are routed to for the duration of one call."""
from __future__ import annotations

import contextlib
from typing import Callable, Dict, Optional, Tuple

import torch
import torch.nn.functional as F

from oracle import macaw_oracle as O

MaskFn = Callable[[str, int, int], torch.Tensor]  # (module name inside model.llm, rows, cols) -> multipliers


class LoraLinear:
    """An adapted weight in the oracle's state dict."""

    def __init__(self, name: str, W, A, B, scaling: float, mask_fn: Optional[MaskFn] = None):
        self.name, self.W, self.A, self.B, self.s, self.mask_fn = name, W, A, B, float(scaling), mask_fn

    def __call__(self, x: torch.Tensor) -> torch.Tensor:
        xd = x
        if self.mask_fn is not None:
            K = x.shape[-1]
            xd = x * self.mask_fn(self.name, x.numel() // K, K).reshape(x.shape).to(x.dtype)
        return F.linear(x, self.W) + self.s * F.linear(F.linear(xd, self.A), self.B)


class _Functional:
    """torch.nn.functional with `linear` dispatching LoraLinear weights."""

    def __getattr__(self, name):
        return getattr(F, name)

    @staticmethod
    def linear(x, w, b=None):
        if isinstance(w, LoraLinear):
            assert b is None
            return w(x)
        return F.linear(x, w, b)


@contextlib.contextmanager
def _lora_linears():
    prev = O.F
    O.F = _Functional()
    try:
        yield
    finally:
        O.F = prev


def llama_forward(embeds, attention_mask, sd: Dict[str, torch.Tensor], hp: dict,
                  adapters: Dict[str, Tuple[torch.Tensor, torch.Tensor, float]], mask_fn: Optional[MaskFn] = None,
                  dtype=torch.float64) -> torch.Tensor:
    """The oracle's llama_forward with LoRA adapters {name inside model.llm: (A, B, scaling)} (unmerged formula)."""
    merged = {k: (v.detach().cpu().to(dtype) if v.is_floating_point() else v) for k, v in sd.items()}
    for name, (A, B, s) in adapters.items():
        merged[f"llm.{name}.weight"] = LoraLinear(name, merged[f"llm.{name}.weight"], A.cpu().to(dtype), B.cpu().to(dtype),
                                                  s, mask_fn)
    with _lora_linears():
        return O.llama_forward(embeds.to(dtype), attention_mask, O._SD(merged, dtype, keep_graph=True), hp)


def loss_and_grads(inputs: dict, sd: Dict[str, torch.Tensor], hp: dict,
                   adapters: Dict[str, Tuple[torch.Tensor, torch.Tensor, float]], mask_fn: Optional[MaskFn] = None,
                   dtype=torch.float32):
    """Loss of MM_LLMs.forward with LoRA adapters on a frozen decoder and its autograd gradients w.r.t. every adapter
    (keys llm.<name>.lora_{A,B}.weight) and every alignment module, as O.full_loss_and_grads does for the full model
    (attention dropout off; the adapters' input dropout given by mask_fn).  -> (loss, {name: grad})."""
    merged, leaves = {}, {}
    for k, v in sd.items():
        if not v.is_floating_point():
            merged[k] = v
            continue
        t = v.detach().cpu().to(dtype)
        if k.startswith(O.ALIGN_PREFIXES):
            t = t.clone().requires_grad_(True)
            leaves[k] = t
        merged[k] = t
    for name, (A, B, s) in adapters.items():
        a = A.detach().cpu().to(dtype).clone().requires_grad_(True)
        b = B.detach().cpu().to(dtype).clone().requires_grad_(True)
        leaves[f"llm.{name}.lora_A.weight"], leaves[f"llm.{name}.lora_B.weight"] = a, b
        merged[f"llm.{name}.weight"] = LoraLinear(name, merged[f"llm.{name}.weight"], a, b, s, mask_fn)
    embeds, mask, labels = O.prepare_inputs(inputs, merged, hp, dtype, keep_graph=True)
    with _lora_linears():
        logits = O.llama_forward(embeds, mask, O._SD(merged, dtype, keep_graph=True), hp)
    loss = O.shifted_ce(logits, labels)
    loss.backward()
    return loss.detach(), {k: v.grad for k, v in leaves.items()}
