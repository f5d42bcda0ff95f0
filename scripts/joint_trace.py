"""Record every C ABI call the gated joint's training, alignment and MBR paths make, and what they compute, for comparing two builds.

    python scripts/joint_trace.py --out DIR
    python scripts/joint_trace.py --compare NEW_DIR OLD_DIR [OLD_RERUN_DIR ...]

--out replaces ``pika_b200.kernels.lib`` with a recording proxy (every wrapper in kernels.py looks ``lib`` up as a module global, so
the proxy sees every call the engine and the MBR trainer make) and runs seeded workloads at the small fixture shapes (V = 40, whose
fc2 takes the row log-sum-exp epilogue, and V = 43, whose logits carry padding columns):
JointFn forward and backward; transducer_loss in bf16 (compacted gradient rows), in fp32-class mode (dense gradient), with
engine._COMPACT_GRAD off and with engine._FUSED_LSE off; transducer_loss_pruned plain, smoothed and with FastEmit and the delay
penalty; transducer_align dense and pruned; one mbr_forward_backward step in bf16 and in fp32-class mode on tests/golden/mbr_small.npz.
Each call is recorded as its entry point and its non-pointer arguments; a pointer argument (by the binding's ``argtypes``) only as
NULL or not, and a ``pk_gemm_desc`` as every field, pointers again as NULL or not.  DIR gets trace.json and results.npz (every cost,
alignment output and parameter ``.grad``).

--compare checks that two traces are equal entry for entry and lists the tensors of results.npz that are not equal bit for bit.  With
reruns of the old build, each differing tensor is also checked against the old build's own run-to-run differences: one that differs
between NEW and OLD but never between OLD and a rerun is a finding.  Exit code 0 when the traces are equal and no
such finding exists.  Needs a GPU for --out.
"""
import argparse
import ctypes
import json
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))


def _field(v, t):
    if t is ctypes.c_void_p:
        return "NULL" if not v else "ptr"
    if isinstance(v, ctypes.Structure):
        return {n: _field(getattr(v, n), ft) for n, ft in v._fields_}
    if isinstance(v, ctypes.Array):
        return [_field(x, v._type_) for x in v]
    return v


class _Recorder:
    def __init__(self, lib):
        self._lib, self.calls = lib, []

    def __getattr__(self, name):
        fn = getattr(self._lib, name)
        types_ = fn.argtypes or []

        def call(*args):
            rec = [name]
            for t, a in zip(types_, args):
                if isinstance(a, ctypes.Structure):
                    rec.append(_field(a, type(a)))
                elif t is ctypes.c_void_p:
                    rec.append("NULL" if not a else "ptr")
                else:
                    rec.append(a)
            self.calls.append(rec)
            return fn(*args)
        return call


def _net(V, reinit=None):
    from pika_b200.model.transducer import Net, add_simple_joiner
    torch.manual_seed(777)
    margs = types.SimpleNamespace(rnn_size=1024, local_rank=0, decoder_type="rnn", brnn=True, encoder_type="transformer",
                                  embd_dim=100, padding_idx=V, dropout=0.2, dec_layers=2, enc_layers=9)
    m = Net(margs, 240, V)
    add_simple_joiner(m, 1024, V)
    if reinit is not None:
        reinit(m)
    return m.cuda().train()


def _grads(out, tag, model):
    for k, p in model.named_parameters():
        if p.grad is not None:
            out["%s/grad/%s" % (tag, k)] = p.grad.detach().float().cpu().numpy()
        p.grad = None


def workloads(out, trace, rec):
    from pika_b200 import engine
    from pika_b200.trainer.mbr import mbr_forward_backward
    d = np.load(os.path.join(ROOT, "tests", "golden", "model_small.npz"))
    x = torch.from_numpy(d["x"]).cuda()
    y = torch.from_numpy(d["y"]).long().cuda()
    tl, ul = torch.from_numpy(d["tlens"]).cuda(), torch.from_numpy(d["ulens"]).cuda()

    def run(tag, prec, fn):
        engine.set_precision(prec)
        engine.set_seed(0x5EED)
        rec.calls = []
        fn(tag)
        torch.cuda.synchronize()
        trace[tag] = rec.calls
        engine.set_precision("bf16")

    for V in (40, 43):
        m = _net(V)

        def joint_fn(tag):
            lp = engine.transducer_forward(m, x, y)
            w = torch.randn(lp.shape, generator=torch.Generator(device="cuda").manual_seed(5), device="cuda")
            (lp * w).sum().backward()
            out[tag + "/lp"] = lp.detach().cpu().numpy()
            _grads(out, tag, m)

        def loss(tag, **kw):
            costs = engine.transducer_loss(m, x, y, tl, ul, **kw)
            costs.sum().backward()
            out[tag + "/costs"] = costs.detach().cpu().numpy()
            _grads(out, tag, m)

        def pruned(tag, **kw):
            s, p = engine.transducer_loss_pruned(m, x, y, tl, ul, 3, 0.5, 1.0, **kw)
            (0.5 * s.sum() + p.sum()).backward()
            out[tag + "/simple"], out[tag + "/pruned"] = s.detach().cpu().numpy(), p.detach().cpu().numpy()
            _grads(out, tag, m)

        def align(tag, **kw):
            for k, v in zip(("frames", "viterbi", "loglik"), engine.transducer_align(m, x, y, tl, ul, **kw)):
                out["%s/%s" % (tag, k)] = v.cpu().numpy()

        for prec in ("bf16", "fp32"):
            run("V%d/%s/joint_fn" % (V, prec), prec, joint_fn)
            run("V%d/%s/loss" % (V, prec), prec, loss)
            run("V%d/%s/loss_reg" % (V, prec), prec, lambda t: loss(t, fastemit_lambda=0.01, delay_penalty=0.005))
            run("V%d/%s/pruned" % (V, prec), prec, pruned)
            run("V%d/%s/pruned_smoothed" % (V, prec), prec, lambda t: pruned(t, lm_only_scale=0.1, am_only_scale=0.05))
            run("V%d/%s/pruned_reg" % (V, prec), prec, lambda t: pruned(t, fastemit_lambda=0.01, delay_penalty=0.005))
            run("V%d/%s/align" % (V, prec), prec, align)
            run("V%d/%s/align_pruned" % (V, prec), prec, lambda t: align(t, prune_range=3))
        for flag in ("_COMPACT_GRAD", "_FUSED_LSE"):
            setattr(engine, flag, False)
            try:
                run("V%d/bf16/loss_no%s" % (V, flag), "bf16", loss)
            finally:
                setattr(engine, flag, True)
        del m

    from fixture_utils import decode_fixture_reinit
    dm = np.load(os.path.join(ROOT, "tests", "golden", "mbr_small.npz"))
    dd = np.load(os.path.join(ROOT, "tests", "golden", "decode_small.npz"))
    m = _net(40, decode_fixture_reinit)
    ret = {"predictions": [[[int(t) for t in h if t != -2] for h in row] for row in dm["hyps"]],
           "scores": [[float(s) for s in row] for row in dm["scores"]]}
    xm, tlm = torch.from_numpy(dd["x"]).cuda(), torch.from_numpy(dd["tlens"]).int().cuda()
    target, ulm = torch.from_numpy(dm["target"]).cuda(), torch.from_numpy(dm["ulens"]).int().cuda()

    def mbr(tag):
        mbr_loss, costs = mbr_forward_backward(m, xm, target, tlm, ulm, ret, blk=0, rnnt_scale=0.5, sm_scale=0.8)
        out[tag + "/mbr_loss"] = np.array(mbr_loss, np.float64)
        out[tag + "/costs"] = costs.detach().cpu().numpy()
        _grads(out, tag, m)

    for prec in ("bf16", "fp32"):
        run("mbr/%s" % prec, prec, mbr)


def record(out_dir):
    from pika_b200 import engine, kernels
    rec = _Recorder(kernels.lib)
    kernels.lib = rec
    engine.set_dropout_enabled(False)
    out, trace = {}, {}
    try:
        workloads(out, trace, rec)
    finally:
        kernels.lib = rec._lib
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "trace.json"), "w") as f:
        json.dump(trace, f)
    np.savez(os.path.join(out_dir, "results.npz"), **out)
    print("joint_trace: %d workloads, %d calls, %d tensors -> %s" % (len(trace), sum(len(v) for v in trace.values()), len(out), out_dir))


def _differs(a, b):
    return a.shape != b.shape or a.tobytes() != b.tobytes()


def compare(new, old, *reruns):
    tn, to = (json.load(open(os.path.join(p, "trace.json"))) for p in (new, old))
    ok = list(tn) == list(to)
    if not ok:
        print("workloads differ: %s vs %s" % (list(tn), list(to)))
    for k in tn:
        a, b = tn[k], to.get(k, [])
        bad = next((i for i, (x, y) in enumerate(zip(a, b)) if x != y), None)
        if bad is None and len(a) != len(b):
            bad = min(len(a), len(b))
        if bad is not None:
            ok = False
            print("trace %s: %d vs %d calls, first difference at call %d:\n  new %s\n  old %s"
                  % (k, len(a), len(b), bad, a[bad] if bad < len(a) else None, b[bad] if bad < len(b) else None))
        else:
            print("trace %s: %d calls, equal" % (k, len(a)))
    rn, ro = np.load(os.path.join(new, "results.npz")), np.load(os.path.join(old, "results.npz"))
    if sorted(rn.files) != sorted(ro.files):
        print("result tensors differ: %s" % sorted(set(rn.files) ^ set(ro.files)))
        ok = False
    noisy = set()
    for r in reruns:
        rr = np.load(os.path.join(r, "results.npz"))
        noisy |= {k for k in ro.files if k in rr.files and _differs(ro[k], rr[k])}
    diff = [k for k in rn.files if k in ro.files and _differs(rn[k], ro[k])]
    for k in diff:
        ok = ok and k in noisy
        print("tensor %s differs (max |diff| %.3g); %s" % (k, float(np.abs(rn[k].astype(np.float64) - ro[k].astype(np.float64)).max()),
                                                           "also between old runs" if k in noisy else "NOT between old runs"))
    print("%d of %d tensors bit-identical; %d differ between old runs; %s"
          % (len(rn.files) - len(diff), len(rn.files), len(noisy), "OK" if ok else "FINDINGS"))
    return ok


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--out")
    ap.add_argument("--compare", nargs="+", metavar="DIR")
    a = ap.parse_args()
    if a.compare:
        sys.exit(0 if compare(*a.compare) else 1)
    record(a.out)


if __name__ == "__main__":
    main()
