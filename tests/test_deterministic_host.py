"""CPU checks of the deterministic rows trainer (DESIGN.md §4.13): the command line's --deterministic option, the
configurations train_cbow rejects before touching a device, and the C ABI's tile-workspace size and argument checks."""
import numpy as np
import pytest

from tests import helpers


def test_command_line_deterministic_option(capsys):
    from g2vec_b200 import cli
    base = ["e.tsv", "c.tsv", "n.tsv", "out"]
    assert cli.parse_arguments(base).deterministic is False
    assert cli.parse_arguments(base + ["--deterministic"]).deterministic is True
    args = cli.parse_arguments(base + ["--deterministic", "--batch", "64", "--reshuffle", "--optimizer", "sgd"])
    assert args.deterministic and args.batch == 64 and args.reshuffle
    assert cli.parse_arguments(base + ["--deterministic", "--algo", "rank1"]).deterministic is True
    with pytest.raises(SystemExit):
        cli.parse_arguments(base + ["--deterministic", "--algo", "rank1", "--batch", "64"])
    assert "--deterministic with --algo rank1 needs a full batch" in capsys.readouterr().err


def test_train_cbow_rejects_rank1_minibatches_and_several_ranks(monkeypatch):
    import g2vec_b200 as g2v
    from g2vec_b200 import cbow
    rowptr, gene, label = helpers.random_windows(50, 20, 1, 5, seed=0)
    args = (rowptr, gene, label, 20, 8, 0.005)
    with pytest.raises(ValueError, match="rank1"):
        g2v.train_cbow(*args, log=None, algo="rank1", batch=16, deterministic=True)

    class TwoRanks:                       # a process group of two; any collective would fail on this object
        def get_world_size(self):
            return 2

        def get_rank(self):
            return 0
    monkeypatch.setattr(cbow, "_dist", lambda: TwoRanks())
    with pytest.raises(ValueError, match="one GPU"):
        g2v.train_cbow(*args, log=None, deterministic=True)


def test_workspace_bytes_follow_the_tile_model():
    from g2vec_b200 import _capi
    lib = _capi.load()
    T = 64
    for n, D in ((0, 128), (1, 128), (256, 128), (257, 100), (150_000, 128), (1_600_000, 512)):
        tiles = -(-n // T)
        want = (-(-8 * tiles // 256) * 256) + 4 * tiles * D
        assert lib.g2v_cbow_det_workspace_bytes(n, D) == want, (n, D)
    assert lib.g2v_cbow_det_workspace_bytes(-1, 128) == 0
    assert lib.g2v_cbow_det_workspace_bytes(10, 0) == 0


def test_entry_points_reject_bad_arguments_before_any_launch():
    from g2vec_b200 import _capi
    lib = _capi.load()
    a = np.zeros(16, np.int64)
    p = a.ctypes.data
    # unknown reduce, negative max_ctas, null workspace
    assert lib.g2v_cbow_fwd_do_det(p, p, p, p, 4, 0.25, p, p, p, p, p, p, 10, 8, 7, p, 0, None) == 2
    assert b"unknown reduce" in lib.g2v_last_error()
    assert lib.g2v_cbow_fwd_do_det(p, p, p, p, 4, 0.25, p, p, p, p, p, p, 10, 8, 0, p, -1, None) == 2
    assert lib.g2v_cbow_fwd_do_det(p, p, p, p, 4, 0.25, p, p, p, p, p, p, 10, 8, 0, None, 0, None) == 2
    assert b"null pointer" in lib.g2v_last_error()
    assert lib.g2v_cbow_fwdbwd_csc_det(p, p, p, p, 4, 0.25, p, p, None, p, p, p, p, p, p, 10, 8, 0, p, 0, None) == 2
    assert lib.g2v_cbow_loop_tail_det(None, p, p, p, p, 4, 0.25, p, p, p, p, None, 10, 8, 0, p, 0, None) == 2
    assert lib.g2v_cbow_batch_expand(p, p, p, p, 11, p, p, 10, 8, 0, None) == 2        # more rows than genes
    assert lib.g2v_cbow_batch_expand(None, p, p, p, 3, p, p, 10, 8, 0, None) == 2
    # empty lists launch nothing
    assert lib.g2v_cbow_fwd_do_det(None, None, None, None, 0, 1.0, None, None, None, None, None, None, 10, 8, 0, None,
                                   0, None) == 0
    assert lib.g2v_cbow_batch_expand(None, None, None, None, 0, None, None, 10, 8, 0, None) == 0
