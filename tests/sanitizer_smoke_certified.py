"""Every branch of the certified accuracy pass (g2v_cbow_eval_certified) once -- D = 128, 256, 512 and the generic
kernel, decided and gathered windows, the forced gather -- and a full-batch run whose chunks replay as CUDA graphs,
meant to be executed under compute-sanitizer on a GPU box, like tests/sanitizer_smoke.py:

    compute-sanitizer --tool memcheck  python tests/sanitizer_smoke_certified.py
    compute-sanitizer --tool racecheck python tests/sanitizer_smoke_certified.py

(not a pytest test).  Each count is checked against g2v_cbow_eval's."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    import torch
    import g2vec_b200 as g2v
    from g2vec_b200 import _capi
    from tests import helpers
    lib = _capi.load()
    st = torch.cuda.current_stream().cuda_stream
    V, N = 300, 700
    rowptr, gene, label = helpers.random_windows(N, V, 0, 40, seed=5)      # includes empty windows
    cu = lambda a, dt=torch.int32: torch.from_numpy(a).to("cuda", dt)
    rp, ge, la = cu(rowptr), cu(gene), cu(label, torch.uint8)
    for D in (128, 256, 512, 40):
        W0, Wo0 = helpers.init_weights(V, D, 1)
        W, Wo = cu(W0, torch.float32), cu(Wo0, torch.float32)
        acc = torch.zeros(4, dtype=torch.int64, device="cuda")
        scratch = torch.empty(2 * V, device="cuda")
        _capi.check(lib.g2v_cbow_eval(rp.data_ptr(), ge.data_ptr(), la.data_ptr(), None, 0, N, W.data_ptr(),
                                      Wo.data_ptr(), acc.data_ptr(), V, D, 0, st), "g2v_cbow_eval")
        for force in (0, 1):
            _capi.check(lib.g2v_cbow_eval_certified(rp.data_ptr(), ge.data_ptr(), la.data_ptr(), None, 0, N,
                                                    W.data_ptr(), Wo.data_ptr(), scratch.data_ptr(),
                                                    acc.data_ptr() + 8 * (1 + force), acc.data_ptr() + 24, V, D, 0,
                                                    force, st), "g2v_cbow_eval_certified")
        a = acc.cpu().tolist()
        assert a[0] == a[1] == a[2], (D, a)
    W0, Wo0 = helpers.init_weights(V, 40, 1)
    _, info = g2v.train_cbow(rowptr, gene, label, V, 40, 0.05, max_epoch=11, seed=0, W_ih0=W0, W_ho0=Wo0, log=None,
                             early_stop=False, return_info=True)
    assert info["graph"]
    print("certified sanitizer smoke OK")


if __name__ == "__main__":
    main()
