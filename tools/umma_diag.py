"""GPU diagnostic: the wgmma conv kernels vs the SIMT kernels on the same engine inputs (python tools/umma_diag.py [frames] [tc]).
Prints rel-L2 per layer (forward and data-gradient) and, on mismatch, where the error sits."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "action-detection_b200")):
    sys.path.insert(0, p)
import torch
from oracle import ssn_oracle as O, synth
from ssn_b200 import _lib
from ssn_b200.engine import BackboneEngine


def rel(a, b):
    return float((a.double() - b.double()).norm() / (b.double().norm() + 1e-30))


def main():
    Fn = int(sys.argv[1]) if len(sys.argv) > 1 else 18
    # mode "tc": SSNB_EXACT_TC (split-operand wgmma) against the fp32 SIMT kernels, bar 2e-5; default: FAST vs SIMT fp16
    tc = len(sys.argv) > 2 and sys.argv[2] == "tc"
    prec, bar = (_lib.EXACT_TC, 2e-5) if tc else (_lib.FAST_FP16, 2e-3)
    dev = torch.device("cuda:0")
    bb = synth.synth_backbone(3, seed=0, calib_frames=2)
    names = [n for (n, *_r) in O.conv_layers(3)]
    spec = {n: (ci, co, k, s, p) for (n, ci, co, k, s, p) in O.conv_layers(3)}

    def make(disable):
        os.environ["SSNB_DISABLE_UMMA"] = "1" if disable else "0"
        e = BackboneEngine(3, Fn, prec, True, 1024.0, dev)
        e.pack([bb[n + ".weight"].to(dev) for n in names], [bb[n + ".bias"].to(dev) for n in names],
               [bb[n + "_bn.weight"].to(dev) for n in names], [bb[n + "_bn.bias"].to(dev) for n in names],
               [bb[n + "_bn.running_mean"].to(dev) for n in names], [bb[n + "_bn.running_var"].to(dev) for n in names])
        return e

    simt, umma = make(True), make(False)
    grads = {}
    for e in (simt, umma):
        dw = [torch.zeros(bb[n + ".weight"].shape, device=dev) for n in names]
        db = [torch.zeros(bb[n + ".bias"].shape, device=dev) for n in names]
        e.bind_grads(dw, db)
        grads[id(e)] = (dw, db)
    g = torch.Generator().manual_seed(1)
    bad = 0
    for i, (kind, iname, oname) in enumerate(umma.ops()):
        if kind != "conv":
            continue
        ci, co, k, s, p = spec[oname[:-3]]
        c, h, w = umma.value_shape(iname)
        x = torch.randn(Fn, c, h, w, generator=g).to(dev)
        for e in (simt, umma):
            e.write(iname, x)
            e.run_op(i, False)
        try:
            torch.cuda.synchronize()
        except Exception as ex:
            print("FWD %s: CUDA error %s" % (oname, ex)); return
        a, b = umma.read(oname), simt.read(oname)
        r = rel(a, b)
        tag = "ok " if r < bar else "BAD"
        print("%s fwd   %-34s cin %4d cout %4d k%d hw %3d  rel %.3e" % (tag, oname, ci, co, k, h, r))
        if r >= bar:
            bad += 1
            d = (a - b).abs()
            print("    err by 16-ch group:", [round(float(d[:, j:j + 16].mean()), 4) for j in range(0, co, 16)][:24])
            print("    err by frame:", [round(float(d[f].mean()), 4) for f in range(min(Fn, 8))])
            print("    err by row y (frame0):", [round(float(d[0, :, y].mean()), 4) for y in range(min(h, 14))])
            print("    err by col x (frame0):", [round(float(d[0, :, :, xx].mean()), 4) for xx in range(min(w, 14))])
            print("    ref mean abs", float(b.abs().mean()), "got mean abs", float(a.abs().mean()))
        # data gradient
        co_, ho, wo = umma.value_shape(oname)
        gy = torch.randn(Fn, co_, ho, wo, generator=g).to(dev) * 0.01
        y = torch.rand(Fn, co_, ho, wo, generator=g).to(dev)
        for e in (simt, umma):
            e.write(oname, y)
            e.write(oname, gy, grad=True)
            e.write(iname, torch.zeros(Fn, c, h, w, device=dev), grad=True)
            e.run_op(i, True)
        try:
            torch.cuda.synchronize()
        except Exception as ex:
            print("DGRAD %s: CUDA error %s" % (oname, ex)); return
        a, b = umma.read(iname, grad=True), simt.read(iname, grad=True)
        r = rel(a, b)
        tag = "ok " if r < bar else "BAD"
        print("%s dgrad %-34s rel %.3e" % (tag, oname, r))
        if r >= bar:
            bad += 1
        ci_ = names.index(oname[:-3])
        a, b = grads[id(umma)][0][ci_], grads[id(simt)][0][ci_]
        r = rel(a, b)
        wbar = 2e-4 if tc else bar        # tc: two fp32 reductions over F*H*W pixels in different orders (both ~1e-5 from exact at F=160)
        tag = "ok " if r < wbar else "BAD"
        print("%s wgrad %-34s rel %.3e  |ref| %.3e |got| %.3e" % (tag, oname, r, float(b.abs().mean()), float(a.abs().mean())))
        if r >= wbar:
            bad += 1
            d = (a - b).abs()
            print("    err by tap:", [round(float(d[:, :, t // k, t % k].mean() / (b.abs().mean() + 1e-30)), 3) for t in range(k * k)])
            print("    err by co/16:", [round(float(d[j:j + 16].mean() / (b.abs().mean() + 1e-30)), 3) for j in range(0, co, 16)][:24])
            print("    err by ci/16:", [round(float(d[:, j:j + 16].mean() / (b.abs().mean() + 1e-30)), 3) for j in range(0, ci, 16)][:40])
    print("umma_diag: %d mismatching launches" % bad)


if __name__ == "__main__":
    main()
