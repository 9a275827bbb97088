"""`train_batch` with the reference's signature and control flow (ml_mdm/trainer.py:13-97, both the fp32 branch and
the `args.fp16` branch the shipped cc12m_1024x1024.yaml selects), using the fused clip + Adam + EMA + zero-grad
sweep when the optimizer is `mdm_b200.optim.FusedAdam` and the reference's separate calls otherwise.

`args.fp16` in the reference means "Using fp16 to speed-up training": get_loss under bf16 autocast, then GradScaler
around the backward and the step (trainer.py:29-61). That branch does the same: the loss is computed inside
torch.autocast("cuda", dtype=torch.bfloat16), which the native denoiser honours by running its weight products on the
weights' hi fp16 plane only (models/native.py autocast_active; its backward follows the forward's mode), and it keeps
the reference's control flow -- loss * loss_factor, the division by num_grad_accumulations before backward, a NaN loss
that neither steps the optimizer nor the scheduler, clipping over model.model.parameters(), GradScaler
scale/unscale/step/update when a scaler is passed."""
import numpy as np
import torch
import torch.nn as nn

from .optim import FusedAdam


def train_batch(model, sample, optimizer, scheduler, logger, args, grad_scaler=None, accumulate_gradient=False,
                num_grad_accumulations=1, ema_model=None, loss_factor=1.0):
    model.train()
    lr = scheduler.get_last_lr()[0]
    if getattr(args, "fp16", False):
        return _train_batch_fp16(model, sample, optimizer, scheduler, logger, args, grad_scaler, accumulate_gradient,
                                 num_grad_accumulations, ema_model, loss_factor, lr)
    losses, times, x_t, means, targets, weights = model.get_loss(sample)
    if weights is None:
        loss = losses.mean()
    else:
        loss = (losses * weights).sum() / weights.sum()
    loss_val = loss.item()
    if np.isnan(loss_val):  # trainer.py:69-74
        optimizer.zero_grad()
        optimizer.step()
        scheduler.step()
        return loss_val, losses, times, x_t, means, targets

    loss.backward()
    # (the reference divides `loss` by num_grad_accumulations only after backward, trainer.py:77-78: no effect)
    if not accumulate_gradient:
        vision = getattr(model.model, "module", model.model).vision_model
        if isinstance(optimizer, FusedAdam):
            optimizer.step(max_grad_norm=args.gradient_clip_norm, ema_model=ema_model)
        else:
            nn.utils.clip_grad_norm_(model.parameters(), args.gradient_clip_norm)
            optimizer.step()
            if ema_model is not None:
                ema_model.update(vision)

    if logger is not None and not accumulate_gradient:
        logger.add_scalar("train/Loss", loss_val)
        logger.add_scalar("lr", lr)

    if not accumulate_gradient:
        optimizer.zero_grad()
        scheduler.step()

    return loss_val, losses, times, x_t, means, targets


def _train_batch_fp16(model, sample, optimizer, scheduler, logger, args, grad_scaler, accumulate_gradient,
                      num_grad_accumulations, ema_model, loss_factor, lr):
    """trainer.py:29-61."""
    with torch.autocast("cuda", dtype=torch.bfloat16):
        losses, times, x_t, means, targets, weights = model.get_loss(sample)
        if weights is None:
            loss = losses.mean()
        else:
            loss = (losses * weights).sum() / weights.sum()
        loss = loss * loss_factor
        loss_val = loss.item()
        if np.isnan(loss_val):  # trainer.py:39-41: no optimizer step, no scheduler step
            optimizer.zero_grad()
            return loss_val, losses, times, x_t, means, targets
        if num_grad_accumulations != 1:
            loss = loss / num_grad_accumulations
    scaling = grad_scaler is not None and grad_scaler.is_enabled()
    (grad_scaler.scale(loss) if scaling else loss).backward()
    if not accumulate_gradient:
        vision = getattr(model.model, "module", model.model).vision_model
        fused = isinstance(optimizer, FusedAdam)
        if scaling:
            grad_scaler.unscale_(optimizer)  # in place on .grad (views of the engine's arena)
        if fused:
            before = optimizer.steps
            if scaling:  # GradScaler.step forwards the keyword arguments to optimizer.step unless it found inf/nan
                grad_scaler.step(optimizer, max_grad_norm=args.gradient_clip_norm, ema_model=ema_model)
            else:
                optimizer.step(max_grad_norm=args.gradient_clip_norm, ema_model=ema_model)
            if optimizer.steps == before and ema_model is not None:
                ema_model.update(vision)  # step skipped: the reference still updates the EMA (trainer.py:57-60)
        else:
            nn.utils.clip_grad_norm_(model.model.parameters(), args.gradient_clip_norm)
            if scaling:
                grad_scaler.step(optimizer)
            else:
                optimizer.step()
            if ema_model is not None:
                ema_model.update(vision)
        if scaling:
            grad_scaler.update()
    if logger is not None and not accumulate_gradient:
        logger.add_scalar("train/Loss", loss_val)
        logger.add_scalar("lr", lr)
    if not accumulate_gradient:
        optimizer.zero_grad()
        scheduler.step()
    return loss_val, losses, times, x_t, means, targets
