"""CPU restatement of the training loop's update block and meters (ssn_train.py:213-250,373-415; binary_train.py:170-197,
288-321): the iter_size division, torch 0.3's clip_grad_norm, accuracy() and AverageMeter, in the meter layout of
ssn_b200.meters.StepMeters.  tests/golden/train_loop.npz holds what the reference's own code computes
(oracle/gen_golden_train_loop.py)."""
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
