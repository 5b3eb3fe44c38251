"""Every class-weighted (*_cw) entry point at small size, inside short trainer runs on every route, meant to be
executed under compute-sanitizer on a GPU box, like tests/sanitizer_smoke.py:

    compute-sanitizer --tool memcheck python tests/sanitizer_smoke_class_weight.py

(not a pytest test).  D = 40 takes the generic kernels, D = 128 the float4 ones; the gene-slab route is forced with 3
slabs.  Each bit-reproducible run is repeated and compared bit for bit, and a run with class_weight=(1, 1) against one
without the argument.  It prints the _cw entry points it called, which must be all ten."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    import g2vec_b200 as g2v
    from g2vec_b200 import cbow
    from tests import helpers

    called = set()
    real = cbow.CbowModel._launch

    def launch(self, name, *a):
        if name.endswith("_cw"):
            called.add(name)
        return real(self, name, *a)
    cbow.CbowModel._launch = launch
    V, N = 300, 700
    rowptr, gene, label = helpers.random_windows(N, V, 0, 40, seed=5)
    for D in (40, 128):
        W0, Wo0 = helpers.init_weights(V, D, 1)
        for algo, det, batch, opt, graph in (("rows", True, 0, "adam", True), ("rows", False, 0, "adam", True),
                                             ("rows", False, 0, "adam", False), ("rank1", False, 0, "adam", True),
                                             ("rank1", False, 100, "sgd", False), ("rows", True, 100, "lazy_adam", True),
                                             ("rows", True, 100, "adam", True), ("rows", False, 100, "adam", True),
                                             ("rows", False, 100, "lazy_adam", True), ("slabs", False, 0, "adam", True)):
            if algo == "slabs":
                if D != 128:
                    continue
                os.environ["G2V_CBOW_SLABS"] = "3"
            kw = dict(seed=0, W_ih0=W0, W_ho0=Wo0, log=None, algo="rows" if algo == "slabs" else algo,
                      deterministic=det, batch=batch, optimizer=opt, early_stop=False, max_epoch=11, use_graph=graph)
            a = g2v.train_cbow(rowptr, gene, label, V, D, 0.05, class_weight=(0.37, 1.9), **kw)
            if det or (algo == "rank1" and batch == 0):
                b = g2v.train_cbow(rowptr, gene, label, V, D, 0.05, class_weight=(0.37, 1.9), **kw)
                assert a.tobytes() == b.tobytes(), (D, algo, opt, batch)
                c = g2v.train_cbow(rowptr, gene, label, V, D, 0.05, class_weight=(1, 1), **kw)
                d = g2v.train_cbow(rowptr, gene, label, V, D, 0.05, **kw)
                assert c.tobytes() == d.tobytes() != a.tobytes(), (D, algo, opt, batch)
            os.environ.pop("G2V_CBOW_SLABS", None)
    print("called:", " ".join(sorted(called)))
    assert len(called) >= 9, called
    print("class weight sanitizer smoke OK")


if __name__ == "__main__":
    main()
