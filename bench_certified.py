#!/usr/bin/env python
"""bench_certified.py -- what the certified accuracy pass (g2v_cbow_eval_certified, DESIGN.md §4.16) saves against the
row-gather pass (g2v_cbow_eval) on bench.py's headline workload, on one H100.

    python bench_certified.py --steps K --warmup W [--rounds R]

Workload: the syn10k windows of bench.py's headline (walks -> windows, 10k genes, hidden 128, split seed 1000).
Reported:
  validation  the validation accuracy pass alone: g2v_cbow_eval against g2v_cbow_eval_certified (its collapse included)
              at the initial weights;
  gathered    windows of the validation list the certified pass gathers rows for, at step 0 and after 5, 20 and 50
              trained steps;
  step        one iteration of the device loop as a CUDA graph, both accuracy passes inside (bench.py's `value`), with
              CbowModel.evaluate on each form;
  production  the 5-iteration graph train_cbow replays, divided by 5, on each form.
Both arms live in the same process and are timed alternately, R rounds of K timed steps after W warm-up steps each (CUDA
events on the launching stream, L2 flushed by a 256 MiB write before every timed step).  Reported: the median over the
rounds of each arm's mean, every round's means, and the ratio certified / row_gather.  Prints one JSON line; writes
nothing.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def parse(argv=None):
    p = argparse.ArgumentParser()
    p.add_argument("--steps", type=int, default=10)
    p.add_argument("--warmup", type=int, default=3)
    p.add_argument("--rounds", type=int, default=3)
    a = p.parse_args(argv)
    if a.steps < 1 or a.warmup < 0 or a.rounds < 1:
        p.error("--steps and --rounds must be >= 1, --warmup >= 0")
    return a


def row_gather_evaluate(self, win, slot, win_begin=0, n_win=None):
    """CbowModel.evaluate's rows route as it was before the certified pass: g2v_cbow_eval."""
    n = int((win.shape[0] - win_begin) if n_win is None else n_win)
    self._launch("g2v_cbow_eval", self.rowptr.data_ptr(), self.gene.data_ptr(), self.label.data_ptr(), self._ptr(win),
                 int(win_begin), n, self.W_ih.data_ptr(), self.W_ho.data_ptr(), self.acc.data_ptr() + 8 * slot, self.V,
                 self.D, self.reduce)


def run(args):
    import torch
    import g2vec_b200 as g2v
    from g2vec_b200 import cbow, _capi
    from bench_deterministic import gpu_facts
    from bench_minibatch import headline_windows
    assert torch.cuda.is_available(), "bench_certified.py needs a GPU (no CPU fallback)"
    dev = torch.device("cuda", torch.cuda.current_device())
    lib = _capi.load()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    ev = lambda: torch.cuda.Event(enable_timing=True)
    K, W, R = args.steps, args.warmup, args.rounds
    arms = ("row_gather", "certified")

    def timed(fn, n):
        pairs = []
        for i in range(n):
            flush.fill_(i & 0xFF)
            a, b = ev(), ev()
            a.record(); fn(); b.record()
            pairs.append((a, b))
        torch.cuda.synchronize()
        return [a.elapsed_time(b) for a, b in pairs]

    def alternate(fns, scale=1.0):
        for fn in fns.values():
            timed(fn, max(W, 1))
        means = {k: [] for k in fns}
        for _ in range(R):
            for k, fn in fns.items():
                means[k].append(float(np.mean(timed(fn, K))) / scale)
        out = {k + "_ms": float(np.median(v)) for k, v in means.items()}
        out["rounds_ms"] = means
        out["ratio"] = out["certified_ms"] / out["row_gather_ms"]
        return out

    rowptr, gene, label, V, D, desc = headline_windows(dev)
    tr, va = cbow.split_indices(int(rowptr.shape[0]) - 1, 1000)
    W0, Wo0 = cbow.init_weights(V, D, 0)
    tr_d = torch.from_numpy(tr.astype(np.int32)).to(dev)
    va_d = torch.from_numpy(va.astype(np.int32)).to(dev)
    res = {"config": desc + ", full batch, %d training / %d validation windows" % (len(tr), len(va))}
    st = lambda: torch.cuda.current_stream(dev).cuda_stream

    # ---- the validation pass alone, and the windows it gathers as training goes on
    m = g2v.CbowModel(rowptr, gene, label, V, D, W0, Wo0, lr=0.005)
    m.prepare_csc(tr_d)
    cnt = torch.zeros(3, dtype=torch.int64, device=dev)
    ptrs = (m.rowptr.data_ptr(), m.gene.data_ptr(), m.label.data_ptr(), va_d.data_ptr(), 0, len(va))
    evals = {
        "row_gather": lambda: _capi.check(lib.g2v_cbow_eval(*ptrs, m.W_ih.data_ptr(), m.W_ho.data_ptr(), cnt.data_ptr(),
                                                            V, D, m.reduce, st()), "g2v_cbow_eval"),
        "certified": lambda: _capi.check(lib.g2v_cbow_eval_certified(*ptrs, m.W_ih.data_ptr(), m.W_ho.data_ptr(),
                                                                     m.st.data_ptr(), cnt.data_ptr(), None, V, D,
                                                                     m.reduce, 0, st()), "g2v_cbow_eval_certified")}
    res["validation"] = alternate(evals)
    gathered, done = {}, 0
    for at in (0, 5, 20, 50):
        while done < at:
            m.fwdbwd(tr_d, len(tr)); m.update(); done += 1
        cnt.zero_()
        _capi.check(lib.g2v_cbow_eval(*ptrs, m.W_ih.data_ptr(), m.W_ho.data_ptr(), cnt.data_ptr(), V, D, m.reduce, st()),
                    "g2v_cbow_eval")
        _capi.check(lib.g2v_cbow_eval_certified(*ptrs, m.W_ih.data_ptr(), m.W_ho.data_ptr(), m.st.data_ptr(),
                                                cnt.data_ptr() + 8, cnt.data_ptr() + 16, V, D, m.reduce, 0, st()),
                    "g2v_cbow_eval_certified")
        c = cnt.cpu().tolist()
        assert c[0] == c[1], (at, c)
        gathered[str(at)] = {"windows": c[2], "of": len(va), "rate": c[2] / len(va), "correct": c[0]}
    res["gathered"] = gathered
    del m
    torch.cuda.empty_cache()

    # ---- the device loop as CUDA graphs, evaluate on each form
    n_steps = (W + 1 + 2 * R * K) * 5 + 16
    step, prod, keep = {}, {}, []
    shipped = cbow.CbowModel.evaluate
    for name in arms:
        cbow.CbowModel.evaluate = row_gather_evaluate if name == "row_gather" else shipped
        try:
            m = g2v.CbowModel(rowptr, gene, label, V, D, W0, Wo0, lr=0.005)
            m.prepare_csc(tr_d)
            m.prepare_slabs(tr_d)
            m.prepare_slabs(va_d)
            loop = cbow.DeviceLoop(m, None, tr_d, va_d, len(tr), n_steps, False, snapshot=False)
            loop.attach()
            try:
                for _ in range(max(W, 1)):
                    loop.one(True)
                loop.reset()
                step[name] = loop.capture([True]).replay
                loop.reset()
                prod[name] = loop.capture([False] * 4 + [True]).replay
            finally:
                loop.detach()
        finally:
            cbow.CbowModel.evaluate = shipped
        keep += [m, loop]
    res["step"] = alternate(step)
    res["production"] = alternate(prod, scale=5.0)
    print(json.dumps({"metric": "cbow_certified_eval", "unit": "ms", "lower_is_better": True, "gpu": gpu_facts(),
                      "steps": K, "warmup": W, "rounds": R, "results": res}))


if __name__ == "__main__":
    run(parse())
