"""CPU restatement of the training loop's update block and meters (ssn_train.py:213-250,373-415; binary_train.py:170-197,
288-321): the iter_size division, torch 0.3's clip_grad_norm, accuracy() and AverageMeter, in the meter layout of
ssn_b200.meters.StepMeters.  tests/golden/train_loop.npz holds what the reference's own code computes
(oracle/gen_golden_train_loop.py)."""
import numpy as np
import torch

SSN_METERS = ("act_loss", "comp_loss", "reg_loss", "loss", "act_acc", "fg_acc", "bg_acc")
BINARY_METERS = ("loss", "act_acc", "fg_acc", "bg_acc")


def clip_grad_norm(parameters, max_norm):
    """torch 0.3's torch.nn.utils.clip_grad_norm (L2): per-parameter norms, their squares summed as Python floats, and every
    gradient multiplied in place by max_norm / (total_norm + 1e-6) when that is < 1; returns total_norm"""
    parameters = [p for p in parameters if p.grad is not None]
    total_norm = 0.0
    for p in parameters:
        total_norm += float(p.grad.data.norm(2)) ** 2
    total_norm = total_norm ** 0.5
    clip_coef = max_norm / (total_norm + 1e-6)
    if clip_coef < 1:
        for p in parameters:
            p.grad.data.mul_(clip_coef)
    return total_norm


def update_block(param_groups, model_parameters, iter_size, clip_gradient):
    """the `if i % args.iter_size == 0:` block up to optimizer.step(): returns total_norm (0 without clipping)"""
    if iter_size != 1:
        for g in param_groups:
            for p in g["params"]:
                p.grad /= iter_size
    if clip_gradient is not None:
        return clip_grad_norm(model_parameters, clip_gradient)
    return 0


def accuracy(output, target):
    """top-1 precision in percent as accuracy() computes it, with the lowest class index winning ties (torch.topk leaves
    their order unspecified): fp32 count times the fp32 rounding of 100.0 / batch_size"""
    pred = output.argmax(1)                # the first maximum
    correct = (pred == target).float().sum(0)
    return correct.mul_(100.0 / target.size(0))


def new_meters(names):
    return {k: [0.0, 0.0] for k in names}


def _update(meter, val, n):
    meter[0] += val * n
    meter[1] += n


def update_ssn_meters(meters, losses, raw_act, target, prop_type, batch_size):
    """ssn_train.py:213-233 for one step: losses (act, comp, reg, total), raw_act / target / prop_type of every proposal"""
    for k, v in zip(SSN_METERS[:4], losses.tolist()):
        _update(meters[k], float(torch.tensor(v, dtype=torch.float32)), batch_size)
    sel = ((prop_type == 0) | (prop_type == 2)).nonzero().view(-1)
    _update_acc(meters, raw_act[sel], target[sel])


def update_binary_meters(meters, loss, scores, target, batch_size):
    """binary_train.py:170-180 for one step (plus the accuracy over all rows, which the reference does not print)"""
    _update(meters["loss"], float(loss), batch_size)
    _update_acc(meters, scores, target)


def _update_acc(meters, act, tgt):
    _update(meters["act_acc"], float(accuracy(act, tgt)), act.size(0))
    fg = accuracy(act.view(-1, 2, act.size(1))[:, 0, :].contiguous(), tgt.view(-1, 2)[:, 0].contiguous())
    bg = accuracy(act.view(-1, 2, act.size(1))[:, 1, :].contiguous(), tgt.view(-1, 2)[:, 1].contiguous())
    _update(meters["fg_acc"], float(fg), act.size(0) // 2)
    _update(meters["bg_acc"], float(bg), act.size(0) // 2)


# ---- the device kernels' documented rules, restated in float64 / numpy (tests/test_gpu_update_block.py) ----------------------


def step_schedule(n_micro, iter_size):
    """the reference's loop: loss.backward() on every micro-batch, the update block when i % iter_size == 0, so a step
    after micro-batch 0 alone and then after every iter_size more; True where micro-batch i ends with a step"""
    return [i % iter_size == 0 for i in range(n_micro)]


def top1(scores):
    """ssnb_train_meters' top-1 of every row of a [rows, cols] fp32 array: the highest score, NaN above every number,
    and among equal scores (-0 == +0) and among NaNs the lowest class index"""
    s = np.asarray(scores, np.float32)
    nan = np.isnan(s)
    real = np.where(nan, np.float32(-np.inf), s)
    return np.where(nan.any(1), nan.argmax(1), real.argmax(1)).astype(np.int64)


def meters_update(buf, scores, target, prop_type, losses, loss_n):
    """one ssnb_train_meters call on the fp64 (sum, count) pairs buf [n_losses + 3, 2], in place: the losses, then top-1
    accuracy over the activity rows (prop_type None: every row; else types 0 and 2), the even ones (fg) and the odd ones
    (bg); an odd count leaves the last activity row in the first meter only.  Each accuracy is the fp32 product
    float(correct) * float(100.0 / n) of correct_k.mul_(100.0 / batch_size)"""
    losses = np.asarray(losses, np.float32).reshape(-1)
    for i, v in enumerate(losses):
        buf[i, 0] += float(v) * loss_n
        buf[i, 1] += loss_n
    act = np.ones(len(target), bool) if prop_type is None else np.isin(np.asarray(prop_type), (0, 2))
    ok = top1(np.asarray(scores)[act]) == np.asarray(target)[act]
    m = int(act.sum())
    pairs = m // 2
    for k, (correct, n) in enumerate(((int(ok.sum()), m), (int(ok[0:2 * pairs:2].sum()), pairs),
                                      (int(ok[1:2 * pairs:2].sum()), pairs))):
        if n == 0:
            continue
        val = np.float32(correct) * np.float32(100.0 / n)
        buf[len(losses) + k, 0] += float(val) * n
        buf[len(losses) + k, 1] += n
    return buf


def grad_norm64(flat, grad_mult, extras=()):
    """ssnb_grad_norm in float64: the L2 norm of every flat gradient times grad_mult (their fp32 product, as the kernel
    forms it) plus the extras, undivided; inf when it exceeds the fp32 range"""
    g = (np.asarray(flat, np.float32) * np.float32(grad_mult)).astype(np.float64)
    t = float(np.dot(g, g))
    for e in extras:
        e = np.asarray(e, np.float32).astype(np.float64)
        t += float(np.dot(e, e))
    return t ** 0.5


def clip_coef(norm, max_norm):
    """torch 0.3's clip rule: c = max_norm / (norm + 1e-6) in float64, with max_norm as the fp32 the kernels are passed
    (norm: the device's fp32 norm, or the reference's float64 one); returns c where c < 1, else None (no clipping: a NaN
    norm clips nothing)"""
    c = float(np.float32(max_norm)) / (float(norm) + 1e-6)
    return c if c < 1.0 else None


def clipped_grad(g, grad_mult, c):
    """the gradient ssnb_sgd_step_groups_clipped uses and writes back: g * fl(grad_mult * fl(c)) in fp32 (g * grad_mult
    where c is None); ssnb_grad_clip's extras are clipped_grad(e, 1, c)"""
    gm = np.float32(grad_mult)
    if c is not None:
        gm = np.float32(gm * np.float32(c))
    return np.asarray(g, np.float32) * gm


def sgd64(param, grad, mom, seg_end, seg_lr, seg_wd, momentum, grad_mult, c):
    """one step of ssnb_sgd_step_groups(_clipped) in float64 from fp32 state: every element of segment s (ends seg_end,
    empty segments allowed) takes d = g * m + wd_s * w with m the fp32 multiplier of clipped_grad, buf = momentum * buf + d,
    w -= lr_s * buf.  Returns (param, momentum) as float64 and, per element, the magnitude of the terms each result is
    formed from (the scale of its fp32 rounding errors)"""
    w = np.asarray(param, np.float32).astype(np.float64)
    b0 = np.asarray(mom, np.float32).astype(np.float64)
    n = len(w)
    starts = np.concatenate([[0], np.asarray(seg_end[:-1])])
    sizes = np.asarray(seg_end) - starts
    lr = np.repeat(np.asarray(seg_lr, np.float32).astype(np.float64), sizes)[:n]
    wd = np.repeat(np.asarray(seg_wd, np.float32).astype(np.float64), sizes)[:n]
    gm = float(clipped_grad(np.float32(1.0), grad_mult, c))
    g = np.asarray(grad, np.float32).astype(np.float64) * gm
    d = g + wd * w
    b = float(np.float32(momentum)) * b0 + d
    p = w - lr * b
    b_scale = np.abs(float(np.float32(momentum)) * b0) + np.abs(g) + np.abs(wd * w)
    p_scale = np.abs(w) + lr * b_scale
    return p, b, p_scale, b_scale
