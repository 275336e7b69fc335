"""tests/golden/train_loop.npz from the REAL reference (build container only: python -m oracle.gen_golden_train_loop).

ssn_train.py and binary_train.py are scripts that do not import on Python 3.12 (argparse at import time, torch 0.3 APIs), so
accuracy(), AverageMeter and the update block of train() (`if i % args.iter_size == 0:` up to optimizer.zero_grad()) are
compiled from their own source text with ast -- the reference's code, unedited -- and run on CPU tensors.  The block's
clip_grad_norm is torch 0.3's (oracle/train_loop_oracle.py restates it; today's torch.nn.utils.clip_grad_norm rounds its
coefficient in fp32), its optimiser a torch.optim.SGD whose step() records the gradients it is given."""
import ast
import os
import types

import numpy as np
import torch

from oracle import train_loop_oracle as TL

REF = "/root/reference"
HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(os.path.dirname(HERE), "tests", "golden")


def _top_level(src, names):
    """the source text of the named top-level defs and classes: validate() (`.cuda(async=True)`) does not parse on 3.7+"""
    chunks, cur = [], None
    for line in src.splitlines(keepends=True):
        if line[:1] not in (" ", "\t", "\n", "#", ""):
            cur = line.split("(")[0].split(":")[0].split()[-1] if line.startswith(("def ", "class ")) else None
            chunks.append([cur, ""])
        if chunks:
            chunks[-1][1] += line
    return "".join(text for name, text in chunks if name in names)


def _compile(script):
    src = _top_level(open(os.path.join(REF, script)).read(), ("accuracy", "AverageMeter", "train"))
    body = ast.parse(src).body
    defs = [n for n in body if (isinstance(n, ast.FunctionDef) and n.name == "accuracy")
            or (isinstance(n, ast.ClassDef) and n.name == "AverageMeter")]
    train = [n for n in body if isinstance(n, ast.FunctionDef) and n.name == "train"][0]
    loop = [n for n in train.body if isinstance(n, ast.For)][0]
    block = [n for n in loop.body if isinstance(n, ast.If) and "iter_size" in ast.unparse(n.test)][0]
    ns = {"torch": torch}
    exec(compile(ast.Module(body=defs, type_ignores=[]), script, "exec"), ns)
    return ns, compile(ast.Module(body=[block], type_ignores=[]), script, "exec")


class _RecordingSGD(torch.optim.SGD):
    def step(self, closure=None):
        self.seen = [p.grad.clone() for g in self.param_groups for p in g["params"]]
        return super().step(closure)


def main():
    out = {}
    for script in ("ssn_train.py", "binary_train.py"):
        tag = script.split("_")[0]
        ns, block = _compile(script)
        g = torch.Generator().manual_seed(11 if tag == "ssn" else 12)
        # accuracy() over all rows and the fg / bg halves, fed to AverageMeter as the loop does, three steps
        meters = {k: ns["AverageMeter"]() for k in ("act", "fg", "bg")}
        for step in range(3):
            rows, cols = (2 * (3 + step), 21) if tag == "ssn" else (8 + 2 * step, 2)
            act = torch.randn(rows, cols, generator=g)
            tgt = torch.randint(0, cols, (rows,), generator=g)
            tgt[::2] = act[::2].argmax(1)
            acc = ns["accuracy"](act, tgt)[0]
            fg = ns["accuracy"](act.view(-1, 2, act.size(1))[:, 0, :].contiguous(), tgt.view(-1, 2)[:, 0].contiguous())[0]
            bg = ns["accuracy"](act.view(-1, 2, act.size(1))[:, 1, :].contiguous(), tgt.view(-1, 2)[:, 1].contiguous())[0]
            meters["act"].update(acc.item(), act.size(0))
            meters["fg"].update(fg.item(), act.size(0) // 2)
            meters["bg"].update(bg.item(), act.size(0) // 2)
            p = "%s_acc%d_" % (tag, step)
            out[p + "scores"], out[p + "target"] = act.numpy(), tgt.numpy()
            out[p + "vals"] = np.array([acc.item(), fg.item(), bg.item()], np.float32)
        out[tag + "_meters"] = np.array([[m.sum, m.count] for m in meters.values()], np.float64)
        # the update block: iter_size 1 / 3, no clip, clip above and below the norm; one parameter outside the groups
        for case, (iter_size, clip) in enumerate(((1, None), (3, None), (3, 1e3), (3, 0.5), (1, 0.05))):
            shapes = [(5, 4), (5,), (3, 2, 2), (7,)]
            params = [torch.nn.Parameter(torch.randn(s, generator=g)) for s in shapes]
            grads = [torch.randn(s, generator=g) * 0.3 for s in shapes]
            before = [q.detach().clone() for q in params]
            for q, gr in zip(params, grads):
                q.grad = gr.clone()
            opt = _RecordingSGD([{"params": params[:2], "lr": 0.1, "weight_decay": 5e-4},
                                 {"params": params[2:3], "lr": 0.2, "weight_decay": 0.0}], lr=0.1, momentum=0.9)
            model = types.SimpleNamespace(parameters=lambda: iter(params))
            env = {"i": 0, "args": types.SimpleNamespace(iter_size=iter_size, clip_gradient=clip), "optimizer": opt,
                   "model": model, "clip_grad_norm": TL.clip_grad_norm, "print": lambda *a, **k: None}
            exec(block, env)
            p = "%s_upd%d_" % (tag, case)
            out[p + "cfg"] = np.array([iter_size, np.nan if clip is None else clip], np.float64)
            for j, (gr, q) in enumerate(zip(grads, params)):
                out[p + "grad%d" % j] = gr.numpy()
                out[p + "param%d" % j] = before[j].numpy()
                out[p + "param_after%d" % j] = q.detach().numpy()
            for j, s in enumerate(opt.seen):
                out[p + "seen%d" % j] = s.numpy()
            out[p + "extra_after"] = (params[3].grad.numpy() if params[3].grad is not None else np.zeros(0, np.float32))
            out[p + "total_norm"] = np.float64(env["total_norm"])
    np.savez_compressed(os.path.join(GOLD, "train_loop.npz"), **out)
    print("wrote train_loop.npz:", len(out), "arrays")


if __name__ == "__main__":
    main()
