"""CUDA flat optimizer step: one launch over the whole parameter buffer (csrc/multi_tensor_opt.cu)."""
from __future__ import annotations

import torch

from .cuda_ext import ext


def flat_step(opt, grad_scale: float = 1.0) -> None:
    E = ext()
    fl = opt.flat
    shadow = fl.shadow
    clip = None
    if opt.clip_norm > 0:                   # the norm kernel writes {norm, coef}, the update on the same stream reads coef
        clip = opt.clip_out
        if opt.clip_scratch is None:
            opt.clip_scratch = torch.zeros(E.flat_grad_norm_scratch(fl.grad.numel()), dtype=torch.float64, device=fl.grad.device)
        E.flat_grad_norm(fl.grad, fl.data, clip, opt.clip_scratch, opt.clip_norm, opt.weight_decay, grad_scale, opt.wd_numel)
    if opt.kind == "adam":
        E.flat_adam(fl.data, fl.grad, opt.m, opt.v, shadow, opt.lr, opt.beta1, opt.beta2, opt.eps,
                    opt.weight_decay, grad_scale, opt.step_dev, opt.wd_numel, clip)
    else:
        E.flat_sgd(fl.data, fl.grad, shadow, opt.lr, opt.weight_decay, grad_scale, opt.wd_numel, clip)


def cast_shadow(fl) -> None:
    if fl.shadow is not None:
        ext().cast_bf16(fl.data, fl.shadow)
