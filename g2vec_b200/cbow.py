"""HOT PATH 2, host side: the modified-CBOW trainer behind the reference's call
``compute_genetovec(pathList, n_genes, hidden_size, learning_rate)`` (/root/reference/G2Vec.py:74,
217-286).  The TF1 graph (two matmuls, sigmoid BCE, Adam, accuracy; :231-251) is replaced by the
fused kernels of csrc/g2v_cbow.cu called through the C ABI; this module keeps what the reference
keeps in Python: shuffle + 80/20 split (:219-226), the epoch loop, the log lines and the early stop
(:259-284).

Multi-GPU (one process per GPU, torch.distributed/NCCL): the parameters are replicated, the
training and validation windows are sharded over the ranks, and the dense gradient is all-reduced
once per optimizer step before every rank applies the identical update.
"""
import math
import time

import numpy as np
import torch

from . import _capi


# ------------------------------------------------------------------------------ host-side pieces
def split_indices(n, seed):
    """``np.random.shuffle(pathList)`` then ``pivot = int(len * 0.8)`` (G2Vec.py:219-222), done on an
    index vector with the same legacy MT19937 stream (RandomState(seed).shuffle)."""
    perm = np.arange(n, dtype=np.int64)
    np.random.RandomState(seed).shuffle(perm)
    pivot = int(n * 0.8)
    return perm[:pivot], perm[pivot:]


def truncated_normal(shape, stddev, rng):
    """tf.truncated_normal (G2Vec.py:234-235): N(0, stddev) re-drawn while |x| > 2 stddev."""
    x = rng.standard_normal(size=shape)
    bad = np.abs(x) > 2.0
    while bad.any():
        x[bad] = rng.standard_normal(size=int(bad.sum()))
        bad = np.abs(x) > 2.0
    return (x * stddev).astype(np.float32)


def init_weights(n_genes, hidden, seed):
    rng = np.random.Generator(np.random.PCG64(seed))
    s = 1.0 / math.sqrt(hidden)
    return truncated_normal((n_genes, hidden), s, rng), truncated_normal((hidden,), s, rng)


def shard_by_nnz(idx, lens, world, rank, keep_order=False):
    """Deal window indices to ranks so every rank gets ~equal gather work: sort by length
    (descending, stable) and deal round-robin (SURVEY.md 8e).  ``keep_order`` (mini-batches): deal the
    shuffled list as it is, ``idx[rank::world]``, so that every batch stays a random sample of the list --
    batch b of the N-GPU run is then the same set of windows as batch b of the 1-GPU run."""
    if world == 1:
        return idx
    if keep_order:
        return idx[rank::world]
    order = np.argsort(-lens[idx], kind="stable")
    return idx[order][rank::world]


# ------------------------------------------------------------------------------------ the model
class CbowModel:
    """Parameters + optimizer state + scratch in HBM, and the three kernel calls."""

    def __init__(self, rowptr, gene, label, n_genes, hidden, W_ih0, W_ho0, optimizer="adam", reduce="sum",
                 lr=0.005, beta1=0.9, beta2=0.999, eps=1e-8, device=None, algo="rows", nvl_group=None,
                 deterministic=False, weight_decay=0.0, class_weight=None):
        check_config(algo, optimizer, deterministic, several_gpus=nvl_group is not None, weight_decay=weight_decay,
                     class_weight=class_weight)
        if isinstance(class_weight, str):
            raise ValueError("CbowModel takes class_weight=None or a pair (w0, w1); train_cbow resolves 'balanced'")
        if not torch.cuda.is_available():
            raise RuntimeError("g2vec_b200 needs a CUDA device (H100, sm_90a); there is no CPU fallback")
        self.lib = _capi.load()
        dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        self.device = dev

        def to(a, dt):
            if isinstance(a, torch.Tensor):
                return a.to(device=dev, dtype=dt).contiguous()
            return torch.from_numpy(np.ascontiguousarray(a)).to(device=dev, dtype=dt)

        self.rowptr = to(rowptr, torch.int32)
        self.gene = to(gene, torch.int32)
        self.label = to(label, torch.uint8)
        self.V, self.D = int(n_genes), int(hidden)
        n_flat = self.V * self.D + self.D
        # rows: parameters, Adam state and gradient are flat [W_ih (V*D) | W_ho (D)] allocations.  With a process
        # group (multi-GPU) the parameters and the gradient live in symmetric memory (peer-mapped, NVLS multicast if
        # the fabric has it) and the optimizer step does the gradient exchange itself (g2v_cbow_update_nvl).
        self.nvl = None
        # lazy_adam: TF1 LazyAdam -- only the rows a batch gathered are updated, fused with their per-gene dO sums
        # (g2v_cbow_fwd_do + g2v_cbow_lazy_adam over the batches of prepare_batches); no g_ih is allocated
        self.lazy = optimizer == "lazy_adam"
        # deterministic (DESIGN.md §4.13): every floating-point sum of a rows step in a fixed order -- the tiled forward
        # (g2v_cbow_*_det) on a prepared CSC list or batch plan, never the scatter or the gene slabs
        self.det = bool(deterministic)
        self._det_ws = None
        # (data_ptr, length) of a window list -> its _WindowList; lazy_adam's batch awaiting update(), the batch dO
        self._lists, self._pending, self._dO = {}, None, None
        if algo == "rows" and nvl_group is not None:
            self.nvl = _nvl_setup(nvl_group, n_flat, dev)
        if algo == "rows":
            self.w_flat = self.nvl["w"] if self.nvl else torch.empty(n_flat, dtype=torch.float32, device=dev)
            self.W_ih = self.w_flat[:self.V * self.D].view(self.V, self.D)
            self.W_ho = self.w_flat[self.V * self.D:]
            self.W_ih.copy_(to(W_ih0, torch.float32).reshape(self.V, self.D))
            self.W_ho.copy_(to(W_ho0, torch.float32).reshape(self.D))
        else:
            self.W_ih = to(W_ih0, torch.float32).reshape(self.V, self.D).clone()
            self.W_ho = to(W_ho0, torch.float32).reshape(self.D).clone()
        self.opt = {"adam": _capi.OPT_ADAM_TF1, "sgd": _capi.OPT_SGD, "lazy_adam": _capi.OPT_ADAM_TF1}[optimizer]
        self.reduce = {"sum": _capi.REDUCE_SUM, "mean": _capi.REDUCE_MEAN}[reduce]
        self.lr, self.beta1, self.beta2, self.eps = float(lr), float(beta1), float(beta2), float(eps)
        # decoupled weight decay (DESIGN.md §4.18), fused into every optimizer launch of update(); 0 = off
        self.wd = float(np.float32(weight_decay))
        # class weights (w0, w1) of the training loss as float32 values (DESIGN.md §4.20), folded into dO by every
        # launch that forms it; None = off
        self.cw = class_weight_pair(class_weight)
        z = lambda *s: torch.zeros(*s, dtype=torch.float32, device=dev)
        self.algo = algo
        # rows: scratch of the certified accuracy pass, {s[g], t[g]} per gene (g2v_cbow_eval_certified)
        self.st = z(2 * self.V) if algo == "rows" else None
        if self.lazy:
            self.g_ih, self.g_ho = None, z(self.D)
            self.g_flat = self.g_ho
            self.s = self.c = None
        elif algo == "rows":
            # one allocation [g_ih | g_ho]: a multi-GPU step all-reduces the whole gradient with ONE collective
            self.g_flat = self.nvl["g"].zero_() if self.nvl else z(n_flat)
            self.g_ih = self.g_flat[:self.V * self.D].view(self.V, self.D)
            self.g_ho = self.g_flat[self.V * self.D:]
            self.s = self.c = None
        else:                       # rank-1: s = W_ih.W_ho, c = X^T.dO; no dense gradient
            self.g_ih = None
            self.g_ho = z(int(self.lib.g2v_cbow_r1_scratch_bytes(self.D)) // 4)   # per-block partials of W_ih^T.c
            self.s, self.c = z(self.V), z(self.V)
        self.m_flat = self.v_flat = None
        if self.opt == _capi.OPT_ADAM_TF1 and algo == "rows":
            self.m_flat, self.v_flat = z(n_flat), z(n_flat)
            vd = self.V * self.D
            self.m_ih, self.v_ih = self.m_flat[:vd].view(self.V, self.D), self.v_flat[:vd].view(self.V, self.D)
            self.m_ho, self.v_ho = self.m_flat[vd:], self.v_flat[vd:]
        elif self.opt == _capi.OPT_ADAM_TF1:
            self.m_ih, self.v_ih, self.m_ho, self.v_ho = z(self.V, self.D), z(self.V, self.D), z(self.D), z(self.D)
        else:
            self.m_ih = self.v_ih = self.m_ho = self.v_ho = None
        # [loss_sum (f64 bits), n_correct_train_fwd, n_correct_val, n_correct_train] as 4 x 8 bytes, then the carry
        # slots a DeviceLoop's tail pass fills for the next step: [carried loss_sum (f64 bits), carried n_correct]
        self.acc = torch.zeros(6, dtype=torch.int64, device=dev)
        # Q of the validation-loss pass (evaluate(..., loss=True), DESIGN.md §4.19): an exact uint64 fixed-point sum
        self.q = torch.zeros(1, dtype=torch.int64, device=dev)
        self.t = 0
        # Adam's beta1^t / beta2^t / alpha_t live on the device (TF1's beta*_power variables), advanced by
        # g2v_cbow_adam_tick: no launch of a step depends on a host-side value, so a step can be a CUDA graph
        self.hyper = torch.tensor([1.0, 1.0, 0.0, 0.0], dtype=torch.float32, device=dev)
        # reduce-on-plateau state of g2v_cbow_lr_plateau (set_lr_plateau), else None: the rate is self.lr
        self.plateau = self._plateau_init = None
        if algo == "rank1":
            self._launch("g2v_cbow_r1_prepare", self.W_ih.data_ptr(), self.W_ho.data_ptr(), self.s.data_ptr(), self.V,
                         self.D)

    def _launch(self, name, *args):
        """C ABI entry point ``name`` on the current stream of the model's device, its error raised under its name."""
        rc = getattr(self.lib, name)(*args, self._stream())
        if rc:
            _capi.check(rc, name)

    def _key(self, win):
        return (0, self.rowptr.shape[0] - 1) if win is None else (win.data_ptr(), win.shape[0])

    def prepared(self, win):
        """The _WindowList of what prepare_csc / prepare_slabs / prepare_batches built for the window list ``win``
        (int32 device tensor, or None for every window of the table), else None.  For reading only."""
        return self._lists.get(self._key(win))

    def _record(self, win):
        key = self._key(win)
        return self._lists.setdefault(key, _WindowList(win, key[1]))

    def prepare_csc(self, win):
        """Transpose the incidence of the window list ``win`` (int32 device tensor) once, so that fwdbwd(win, ...)
        over the WHOLE list reduces dO per gene without floating-point atomics: rank1 forms c deterministically,
        rows writes each gradient row once (g2v_cbow_fwdbwd_csc) instead of red.adding a row per (window, gene).
        The windows are static across steps (full batch), so this is setup; calling it again rebuilds."""
        w = win.to(torch.int64)
        starts = self.rowptr[w].to(torch.int64)
        lens = self.rowptr[w + 1].to(torch.int64) - starts
        total = int(lens.sum())
        pos = torch.repeat_interleave(torch.arange(w.shape[0], device=self.device), lens)
        first = torch.cumsum(lens, 0) - lens
        idx = starts[pos] + (torch.arange(total, device=self.device) - first[pos])
        g = self.gene[idx].to(torch.int64)
        g, order = torch.sort(g, stable=True)
        cscptr = torch.zeros(self.V + 1, dtype=torch.int64, device=self.device)
        cscptr[1:] = torch.cumsum(torch.bincount(g, minlength=self.V), 0)
        rec = self._record(win)
        rec.cscptr, rec.pos = cscptr.to(torch.int32), pos[order].to(torch.int32)
        rec.dO = torch.empty(w.shape[0], dtype=torch.float32, device=self.device)

    def prepare_batches(self, win, batch):
        """lazy_adam: cut the window list ``win`` (int32 device tensor) into consecutive batches of ``batch`` windows
        (the last one shorter) and record for every batch the ascending genes it gathers, their segment pointers and
        their positions relative to the batch start -- the transposed incidence of each batch, O(nnz + sum of touched
        genes) in all, built on the device by g2v_cbow_batch_plan.  fwdbwd(win, n, win_begin=lo, n_win=nb) then finds
        batch [lo, lo + nb).  A list has one plan at a time: calling it again for the same list (rewritten in place,
        as a reshuffled epoch is, or with another batch size) replaces the list's plan and releases the buffers of a
        previous batch size.  The buffers are allocated on the first call for a (list, batch size) only, and each
        call reads the per-batch row offsets back once."""
        n = int(win.shape[0])
        B = min(int(batch), n) if batch > 0 else n
        if n == 0:
            return
        rec = self._record(win)
        rec.brp = None
        if rec.plan is None or rec.plan.B != B:
            rec.plan = None
            rec.plan = _PlanBuffers(self, win, B)
        rec.B, rec.brp = B, rec.plan.build(win)[3].tolist()
        if self._dO is None or self._dO.shape[0] < B:
            self._dO = torch.empty(B, dtype=torch.float32, device=self.device)
        self._pending = None

    def batch_touched(self, win, win_begin, n):
        """Number of distinct genes of batch [win_begin, win_begin + n) of a list given to prepare_batches."""
        rec = self.prepared(win)
        rows = rec.batch(win_begin, n) if rec is not None else None
        if rows is None:
            raise KeyError((win_begin, n))
        return rows[1]

    def prepare_slabs(self, win, win_begin=0, n_win=None):
        """rows only, tables larger than the L2 (csrc/g2v_cbow_slab.cu): record once, for the static window list
        ``win`` (int32 device tensor or None), where every window's sorted gene list crosses the gene-slab
        boundaries; fwdbwd()/evaluate() over exactly this list then run slab by slab, L2-resident."""
        if self.algo != "rows" or self.det:
            return False
        import ctypes
        if not hasattr(self, "_n_slabs"):
            s = ctypes.c_int32(1)
            _capi.check(self.lib.g2v_cbow_slab_plan(self.V, self.D, ctypes.byref(s)), "g2v_cbow_slab_plan")
            self._n_slabs = int(s.value)
        n = ((win.shape[0] if win is not None else self.rowptr.shape[0] - 1) - win_begin) if n_win is None else n_win
        if self._n_slabs <= 1 or n <= 0:
            return False
        ws = torch.empty(int(self.lib.g2v_cbow_slab_workspace_bytes(int(n), self.D, self._n_slabs)), dtype=torch.uint8,
                         device=self.device)
        self._launch("g2v_cbow_slab_setup", self.rowptr.data_ptr(), self.gene.data_ptr(), self._ptr(win),
                     int(win_begin), int(n), self.V, self._n_slabs, ws.data_ptr())
        self._record(win).slabs[(int(win_begin), int(n))] = ws
        return True

    def grad_tensors(self):
        """What a multi-GPU step must all-reduce (sum) between fwdbwd() and update(): nothing when update() does
        the exchange itself over NVLink (self.nvl)."""
        if self.nvl:
            return []
        return [self.g_flat] if self.algo == "rows" else [self.c]

    def exchange(self):
        if self.nvl:
            return "nvl-multicast (multimem.ld_reduce / multimem.st)" if self.nvl["g_mc"] else "nvl-p2p (peer loads / stores)"
        return "nccl all_reduce"

    def _stream(self):
        return torch.cuda.current_stream(self.device).cuda_stream

    @staticmethod
    def _ptr(t):
        return 0 if t is None else t.data_ptr()

    def route(self, win, win_begin=0, n_win=None):
        """The route (choose_route) fwdbwd(win, ..., win_begin, n_win) takes; raises as that fwdbwd would."""
        n = (win.shape[0] - win_begin) if n_win is None else n_win
        return choose_route(self.algo, self.lazy, self.det, self.prepared(win), win_begin, n, win is None)

    def fwdbwd(self, win, n_total, win_begin=0, n_win=None):
        """Accumulate the gradient of the listed windows into g_ih / g_ho (loss sum -> acc[0],
        pre-update correct count -> acc[1])."""
        n = (win.shape[0] - win_begin) if n_win is None else n_win
        rec = self._lists.get(self._key(win))
        r = choose_route(self.algo, self.lazy, self.det, rec, win_begin, n, win is None)
        getattr(self, "_fwdbwd_" + r)(win, rec, 1.0 / float(n_total), int(win_begin), int(n))

    def _fwdbwd_scatter(self, win, rec, scale, lo, n):
        name, cw = self._cw("g2v_cbow_fwdbwd")
        self._launch(name, self.rowptr.data_ptr(), self.gene.data_ptr(), self.label.data_ptr(),
                     self._ptr(win), lo, n, scale, self.W_ih.data_ptr(), self.W_ho.data_ptr(), self.g_ih.data_ptr(),
                     self.g_ho.data_ptr(), self.acc.data_ptr(), self.acc.data_ptr() + 8, self.V, self.D, self.reduce,
                     *cw)

    def _fwdbwd_slabs(self, win, rec, scale, lo, n):
        name, cw = self._cw("g2v_cbow_fwdbwd_slabs")
        self._launch(name, self.gene.data_ptr(), self.label.data_ptr(), self._ptr(win), lo, n, scale,
                     self.W_ih.data_ptr(), self.W_ho.data_ptr(), self.g_ih.data_ptr(), self.g_ho.data_ptr(),
                     self.acc.data_ptr(), self.acc.data_ptr() + 8, self.V, self.D, self.reduce, self._n_slabs,
                     rec.slabs[(lo, n)].data_ptr(), *cw)

    def _csc_args(self, win, rec, scale, n):
        return (self.rowptr.data_ptr(), self.gene.data_ptr(), self.label.data_ptr(), win.data_ptr(), n, scale,
                self.W_ih.data_ptr(), self.W_ho.data_ptr(), rec.cscptr.data_ptr(), rec.pos.data_ptr(),
                rec.dO.data_ptr(), self.g_ih.data_ptr(), self.g_ho.data_ptr(), self.acc.data_ptr(),
                self.acc.data_ptr() + 8, self.V, self.D, self.reduce)

    def _fwdbwd_csc(self, win, rec, scale, lo, n):
        name, cw = self._cw("g2v_cbow_fwdbwd_csc")
        self._launch(name, *self._csc_args(win, rec, scale, n), *cw)

    def _fwdbwd_csc_det(self, win, rec, scale, lo, n):
        name, cw = self._cw("g2v_cbow_fwdbwd_csc_det")
        self._launch(name, *self._csc_args(win, rec, scale, n), self.det_workspace(n).data_ptr(), 0, *cw)

    def _fwdbwd_batch_lazy(self, win, rec, scale, lo, n):
        """dO*scale per position of the batch; update() then applies the lazy step to the batch's rows."""
        r0, r1 = rec.brp[lo // rec.B], rec.brp[lo // rec.B + 1]
        self._pending = (rec.plan, r0, r1 - r0)
        self._fwd_do(win, scale, lo, n)

    def _fwdbwd_batch_det(self, win, rec, scale, lo, n):
        r0, n_rows = rec.batch(lo, n)
        self._fwd_do(win, scale, lo, n)
        p = rec.plan
        self._launch("g2v_cbow_batch_expand", p.rows.data_ptr() + 4 * r0, p.segptr.data_ptr() + 4 * r0, p.pos.data_ptr(),
                     self._dO.data_ptr(), n_rows, self.W_ho.data_ptr(), self.g_ih.data_ptr(), self.V, self.D, 0)

    def _fwdbwd_r1(self, win, rec, scale, lo, n):
        name, cw = self._cw("g2v_cbow_r1_windows")
        self._launch(name, self.rowptr.data_ptr(), self.gene.data_ptr(), self.label.data_ptr(),
                     self._ptr(win), lo, n, scale, self.s.data_ptr(), self.c.data_ptr(), self.acc.data_ptr(),
                     self.acc.data_ptr() + 8, self.V, self.reduce, *cw)

    def _fwdbwd_r1_csc(self, win, rec, scale, lo, n):
        name, cw = self._cw("g2v_cbow_r1_windows_csc")
        self._launch(name, self.rowptr.data_ptr(), self.gene.data_ptr(), self.label.data_ptr(),
                     win.data_ptr(), n, scale, self.s.data_ptr(), rec.cscptr.data_ptr(), rec.pos.data_ptr(),
                     rec.dO.data_ptr(), self.c.data_ptr(), self.acc.data_ptr(), self.acc.data_ptr() + 8, self.V,
                     self.reduce, *cw)

    def det_workspace(self, n):
        """The tile workspace of a deterministic forward over n windows (g2v_cbow_det_workspace_bytes), grown on
        demand and shared by every such forward of this model (they run in stream order)."""
        nbytes = int(self.lib.g2v_cbow_det_workspace_bytes(int(n), self.D))
        if self._det_ws is None or self._det_ws.numel() < nbytes:
            self._det_ws = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=self.device)
        return self._det_ws

    def _fwd_do(self, win, scale, lo, n):
        """dO*scale of batch [lo, lo + n) into self._dO, with its loss, count and g_ho (in a fixed order if det)."""
        args = (self.rowptr.data_ptr(), self.gene.data_ptr(), self.label.data_ptr(), win.data_ptr() + 4 * lo, n, scale,
                self.W_ih.data_ptr(), self.W_ho.data_ptr(), self._dO.data_ptr(), self.g_ho.data_ptr(),
                self.acc.data_ptr(), self.acc.data_ptr() + 8, self.V, self.D, self.reduce)
        if self.det:
            name, cw = self._cw("g2v_cbow_fwd_do_det")
            self._launch(name, *args, self.det_workspace(n).data_ptr(), 0, *cw)
        else:
            name, cw = self._cw("g2v_cbow_fwd_do")
            self._launch(name, *args, *cw)

    def loop_tail(self, ctl, win, n_total):
        """A carried DeviceLoop's training-accuracy pass over ``win``, whose fwdbwd routes to csc or csc_det
        (g2v_cbow_loop_tail[_det]): it leaves dO in the list's record, which the next step's fwdbwd expands."""
        rec = self.prepared(win)
        args = (ctl.data_ptr(), self.rowptr.data_ptr(), self.gene.data_ptr(), self.label.data_ptr(), win.data_ptr(),
                rec.n, 1.0 / float(n_total), self.W_ih.data_ptr(), self.W_ho.data_ptr(), rec.dO.data_ptr(),
                self.g_ho.data_ptr(), self.acc.data_ptr(), self.V, self.D, self.reduce)
        if self.det:
            name, cw = self._cw("g2v_cbow_loop_tail_det")
            self._launch(name, *args, self.det_workspace(rec.n).data_ptr(), 0, *cw)
        else:
            name, cw = self._cw("g2v_cbow_loop_tail")
            self._launch(name, *args, *cw)

    def loop_tail_val(self, ctl, win, n_total, va):
        """loop_tail(ctl, win, n_total) and evaluate(va, 2) on the certified pass as one window launch
        (g2v_cbow_loop_tail_val, DESIGN.md §4.32): the same dO, counts and acc[5]; g_ho and acc[4] up to the order of
        their atomics.  For a carried loop whose training list routes to csc and whose D is in TAIL_VAL_D."""
        rec = self.prepared(win)
        name, cw = self._cw("g2v_cbow_loop_tail_val")
        self._launch(name, ctl.data_ptr(), self.rowptr.data_ptr(), self.gene.data_ptr(), self.label.data_ptr(),
                     win.data_ptr(), rec.n, 1.0 / float(n_total), va.data_ptr(), int(va.shape[0]),
                     self.W_ih.data_ptr(), self.W_ho.data_ptr(), self.st.data_ptr(), rec.dO.data_ptr(),
                     self.g_ho.data_ptr(), self.acc.data_ptr(), self.V, self.D, self.reduce, *cw)

    def _lazy_update(self, adev):
        plan, r0, n_rows = self._pending or (None, 0, 0)
        self._pending = None
        name, wd = self._opt("g2v_cbow_lazy_adam")
        self._launch(name, plan.rows.data_ptr() + 4 * r0 if n_rows else None,
                     plan.segptr.data_ptr() + 4 * r0 if n_rows else None, plan.pos.data_ptr() if n_rows else None,
                     self._dO.data_ptr() if n_rows else None, n_rows, self.W_ih.data_ptr(), self.m_ih.data_ptr(),
                     self.v_ih.data_ptr(), self.W_ho.data_ptr(), self.m_ho.data_ptr(), self.v_ho.data_ptr(),
                     self.g_ho.data_ptr(), self.V, self.D, self.lr, self.beta1, self.beta2, self.eps, *wd, self.t, adev)

    def set_lr_plateau(self, patience, factor, min_lr, n_steps):
        """Reduce-on-plateau learning rate (DESIGN.md §4.17): from now on the Adam step size is computed from the rate
        in ``self.plateau`` (g2v_cbow_adam_tick_lr), which lr_decide() cuts by ``factor`` (not below ``min_lr``) after
        ``patience`` steps in a row without a validation count above the best.  The rates of the first ``n_steps``
        decided steps are recorded.  Adam optimizers only."""
        if self.opt != _capi.OPT_ADAM_TF1:
            raise ValueError("the reduce-on-plateau learning rate needs an Adam optimizer")
        cap = max(int(n_steps), 1)
        head = torch.tensor([int(patience), -1, 0, 0, 0, cap, 0, 0], dtype=torch.int64)
        rates = torch.zeros(4 + cap + (cap & 1), dtype=torch.float32)
        rates[:3] = torch.tensor([np.float32(self.lr), np.float32(factor), np.float32(min_lr)])
        self._plateau_init = torch.cat([head, rates.view(torch.int64)])
        self.plateau = self._plateau_init.to(self.device)

    def lr_reset(self):
        """Put the rate state back to its start: best -1, wait 0, no step decided, the initial rate."""
        if self.plateau is not None:
            self.plateau.copy_(self._plateau_init)

    def lr_decide(self, counts_ptr, stride=0, n_decided_ptr=None):
        """g2v_cbow_lr_plateau on the validation counts at ``counts_ptr`` (see include/g2vec_b200.h)."""
        self._launch("g2v_cbow_lr_plateau", self.plateau.data_ptr(), counts_ptr, int(stride), n_decided_ptr)

    def _opt(self, name):
        """The optimizer entry point ``name`` and the arguments it takes between eps and t: its _wd form with the
        model's weight decay, or with weight decay off the plain entry point (the same launches), so that a run
        without decay calls exactly what it called before the option existed."""
        return (name + "_wd", (self.wd,)) if self.wd else (name, ())

    def _cw(self, name):
        """The dO-forming entry point ``name`` and the arguments it takes before the stream: its _cw form with the
        model's class weights (w0, w1), or without class weights the plain entry point, so that a run without them
        calls exactly what it called before the option existed (DESIGN.md §4.20)."""
        return (name + "_cw", self.cw) if self.cw is not None else (name, ())

    def update(self):
        """One optimizer step; every branch decays the elements it updates by the model's weight decay (self.wd, a
        launch constant, DESIGN.md §4.18)."""
        self.t += 1
        adev = 0
        if self.opt == _capi.OPT_ADAM_TF1:
            if self.plateau is not None:
                self._launch("g2v_cbow_adam_tick_lr", self.hyper.data_ptr(), self.plateau.data_ptr() + 64, self.beta1,
                             self.beta2)
            else:
                self._launch("g2v_cbow_adam_tick", self.hyper.data_ptr(), self.lr, self.beta1, self.beta2)
            adev = self.hyper.data_ptr()
        if self.lazy:
            self._lazy_update(adev)
            return
        if self.algo == "rank1":
            name, wd = self._opt("g2v_cbow_r1_update")
            self._launch(name, self.W_ih.data_ptr(), self.W_ho.data_ptr(), self._ptr(self.m_ih),
                         self._ptr(self.v_ih), self._ptr(self.m_ho), self._ptr(self.v_ho), self.c.data_ptr(),
                         self.g_ho.data_ptr(), self.s.data_ptr(), self.V, self.D, self.opt, self.lr, self.beta1,
                         self.beta2, self.eps, *wd, self.t, adev)
            return
        if self.nvl:
            # gradient exchange fused with the optimizer: barrier (every rank's gradient complete) -> reduce-scatter +
            # Adam on the owned slice + all-gather of the new weights in ONE kernel -> barrier (weights delivered)
            nv = self.nvl
            nv["hg"].barrier(channel=0)
            name, wd = self._opt("g2v_cbow_update_nvl")
            self._launch(name, nv["hg"].buffer_ptrs_dev, nv["hw"].buffer_ptrs_dev, nv["g_mc"],
                         nv["w_mc"], self._ptr(self.m_flat), self._ptr(self.v_flat), self.V * self.D + self.D,
                         nv["rank"], nv["world"], self.opt, self.lr, self.beta1, self.beta2, self.eps, *wd, self.t, adev)
            nv["hg"].barrier(channel=1)
            return
        name, wd = self._opt("g2v_cbow_update")
        self._launch(name, self.W_ih.data_ptr(), self.W_ho.data_ptr(), self._ptr(self.m_ih),
                     self._ptr(self.v_ih), self._ptr(self.m_ho), self._ptr(self.v_ho), self.g_ih.data_ptr(),
                     self.g_ho.data_ptr(), self.V, self.D, self.opt, self.lr, self.beta1, self.beta2, self.eps, *wd,
                     self.t, adev)

    def evaluate(self, win, slot, win_begin=0, n_win=None, loss=False):
        """Add the number of correctly classified listed windows into acc[slot].  ``loss``: then also add the windows'
        validation loss Q (g2v_cbow_val_loss, DESIGN.md §4.19) into self.q, from the s = W_ih.W_ho of the weights the
        count was taken at: rank1's s, the certified pass's st, or on the gene-slab route a fresh st."""
        lo = int(win_begin)
        n = int((win.shape[0] - win_begin) if n_win is None else n_win)
        rec = self.prepared(win)
        # the accuracy pass has no backward: it routes as the plain forward does (rank1, or rows with or without slabs)
        r = choose_route(self.algo, False, False, rec, lo, n)
        acc = self.acc.data_ptr() + 8 * slot
        if r in ("r1", "r1_csc"):
            self._launch("g2v_cbow_r1_windows", self.rowptr.data_ptr(), self.gene.data_ptr(), self.label.data_ptr(),
                         self._ptr(win), lo, n, 0.0, self.s.data_ptr(), 0, 0, acc, self.V, self.reduce)
        elif r == "slabs":
            self._launch("g2v_cbow_eval_slabs", self.gene.data_ptr(), self.label.data_ptr(), self._ptr(win), lo, n,
                         self.W_ih.data_ptr(), self.W_ho.data_ptr(), acc, self.V, self.D, self.reduce, self._n_slabs,
                         rec.slabs[(lo, n)].data_ptr())
        else:
            # the count g2v_cbow_eval gives, rows gathered only for windows a float32 bound cannot decide (§4.16)
            self._launch("g2v_cbow_eval_certified", self.rowptr.data_ptr(), self.gene.data_ptr(),
                         self.label.data_ptr(), self._ptr(win), lo, n, self.W_ih.data_ptr(), self.W_ho.data_ptr(),
                         self.st.data_ptr(), acc, None, self.V, self.D, self.reduce, 0)
        if not loss:
            return
        if r in ("r1", "r1_csc"):
            s, stride = self.s, 1
        else:
            if r == "slabs":                     # the slab passes do not write st
                self._launch("g2v_cbow_st_prepare", self.W_ih.data_ptr(), self.W_ho.data_ptr(), self.st.data_ptr(),
                             self.V, self.D)
            s, stride = self.st, 2
        self._launch("g2v_cbow_val_loss", self.rowptr.data_ptr(), self.gene.data_ptr(), self.label.data_ptr(),
                     self._ptr(win), lo, n, s.data_ptr(), stride, self.q.data_ptr(), self.V, self.reduce)

    def loss_sum(self, acc_host):
        return float(acc_host[:1].view(torch.float64)[0])


# the hidden sizes g2v_cbow_loop_tail_val has kernels for
TAIL_VAL_D = (128, 256, 512)

# what early stopping and the reduce-on-plateau rate can decide on (train_cbow's ``monitor``)
MONITORS = ("val_acc", "val_loss")
# the validation-loss pass's fixed point (DESIGN.md §4.19): q_n = rint(min(l_n, LOSS_CAP) * 2^LOSS_BITS), and the
# monitored score 2^62 - Q, non-negative and higher-is-better like a count
LOSS_CAP, LOSS_BITS, SCORE_TOP = 64.0, 24, 1 << 62


def val_loss_mean(Q, n_val):
    """The mean validation loss Q 2^-24 / n_val of an integer Q over n_val windows (0 for none)."""
    return int(Q) / (max(int(n_val), 1) << LOSS_BITS)         # integer true division: correctly rounded


def class_weight_pair(class_weight):
    """The float32 class weights (w0, w1) of a pair of finite numbers > 0 that stay so in float32, as Python floats;
    None for None.  Anything else raises ValueError ("balanced" too: train_cbow resolves it from the labels)."""
    if class_weight is None:
        return None
    msg = ("class_weight must be None, 'balanced' or a pair (w0, w1) of finite numbers > 0 that stay finite and > 0 "
           "in float32 (the weights of the label-0 and label-1 windows in the training loss)")
    if isinstance(class_weight, (str, bytes)) or not hasattr(class_weight, "__len__") or len(class_weight) != 2:
        raise ValueError(msg)
    out = []
    for w in class_weight:
        if isinstance(w, (bool, np.bool_)) or not isinstance(w, (int, float, np.integer, np.floating)):
            raise ValueError(msg)
        with np.errstate(over="ignore", under="ignore"):
            w32 = np.float32(w)
        if not (math.isfinite(float(w32)) and float(w32) > 0.0):
            raise ValueError(msg)
        out.append(float(w32))
    return tuple(out)


def balanced_class_weight(labels, tr):
    """sklearn's compute_class_weight("balanced") on the training split ``tr`` (indices into ``labels``):
    w_y = float32(n_tr / (2 n_tr,y)), computed in float64.  A split without both labels raises ValueError."""
    y = np.asarray(labels.cpu() if isinstance(labels, torch.Tensor) else labels).reshape(-1)[np.asarray(tr, np.int64)]
    n1 = int(np.count_nonzero(y))
    n = int(y.shape[0])
    if n1 == 0 or n1 == n:
        raise ValueError("class_weight='balanced' needs both labels in the training split (it has %d windows of label "
                         "0 and %d of label 1)" % (n - n1, n1))
    return (float(np.float32(n / (2.0 * (n - n1)))), float(np.float32(n / (2.0 * n1))))


def check_config(algo, optimizer, deterministic, several_gpus=False, batch=0, reshuffle=False, patience=1,
                 lr_patience=0, lr_factor=0.1, min_lr=0.0, weight_decay=0.0, monitor="val_acc", class_weight=None):
    """Refuse (ValueError) what train_cbow and CbowModel cannot run, before any device work.  ``several_gpus``: a
    process group of more than one rank; ``batch``, ``reshuffle``, ``patience``, ``lr_patience``, ``lr_factor``,
    ``min_lr``, ``weight_decay``, ``monitor`` and ``class_weight`` as train_cbow takes them."""
    if not (isinstance(class_weight, str) and class_weight == "balanced"):
        class_weight_pair(class_weight)
    if not isinstance(monitor, str) or monitor not in MONITORS:
        raise ValueError("monitor must be 'val_acc' (the correct validation count) or 'val_loss' (the validation "
                         "loss): the value early stopping and the reduce-on-plateau rate decide on")
    if (isinstance(weight_decay, bool) or not isinstance(weight_decay, (int, float, np.integer, np.floating))
            or not 0.0 <= float(np.float32(weight_decay)) < 1.0):
        raise ValueError("weight_decay must be a finite number with 0 <= weight_decay < 1 in float32 (the fraction of "
                         "every weight removed per optimizer step; 0 = off)")
    if isinstance(patience, bool) or not isinstance(patience, (int, np.integer)) or patience < 1:
        raise ValueError("patience must be an int >= 1 (the number of bad epochs in a row that stops the run)")
    if isinstance(lr_patience, bool) or not isinstance(lr_patience, (int, np.integer)) or lr_patience < 0:
        raise ValueError("lr_patience must be an int >= 0 (epochs without improvement before the learning rate is "
                         "cut; 0 = never)")
    if (isinstance(lr_factor, bool) or not isinstance(lr_factor, (int, float, np.integer, np.floating))
            or not 0.0 < float(np.float32(lr_factor)) < 1.0):
        raise ValueError("lr_factor must be a number in (0, 1) (what the learning rate is multiplied by at a plateau)")
    if (isinstance(min_lr, bool) or not isinstance(min_lr, (int, float, np.integer, np.floating))
            or not 0.0 <= float(min_lr) < math.inf):
        raise ValueError("min_lr must be a finite number >= 0 (the learning rate is never cut below it)")
    if lr_patience > 0 and optimizer == "sgd":
        raise ValueError("lr_patience > 0 needs optimizer='adam' or 'lazy_adam': optimizer='sgd' takes its rate from "
                         "the host")
    if algo not in ("rows", "rank1"):
        raise ValueError("algo must be 'rows' (gather/scatter of embedding rows) or 'rank1' (collapsed)")
    if reshuffle and batch <= 0:
        raise ValueError("reshuffle=True needs mini-batches (batch > 0)")
    if deterministic and several_gpus:
        raise ValueError("deterministic=True runs on one GPU only")
    if deterministic and algo == "rank1" and batch > 0:
        raise ValueError("deterministic=True with algo='rank1' needs a full batch: rank1's mini-batch c uses atomics")
    if optimizer == "lazy_adam" and algo != "rows":
        raise ValueError("optimizer='lazy_adam' needs algo='rows' (rank1 keeps s = W_ih.W_ho, which every W_ho step "
                         "changes for every gene)")
    if optimizer == "lazy_adam" and several_gpus:
        raise ValueError("optimizer='lazy_adam' runs on one GPU only")


class _WindowList:
    """What a CbowModel prepared for one window list.  It holds the list (None: every window of the table), so the
    list's address, the model's key for it, cannot be reused for another list while the record exists."""

    def __init__(self, win, n):
        self.win, self.n = win, n
        self.cscptr = self.pos = self.dO = None      # prepare_csc: the whole list's CSC and its dO per list position
        self.slabs = {}                              # prepare_slabs: (win_begin, n_win) -> slab workspace
        self.plan, self.B, self.brp = None, 0, None  # prepare_batches: _PlanBuffers, batch size, row offset per batch

    def whole(self, win_begin, n):
        return self.cscptr is not None and win_begin == 0 and n == self.n

    def batch(self, win_begin, n):
        """(first row, number of rows) of planned batch [win_begin, win_begin + n) in the plan, else None."""
        if self.brp is None or win_begin % self.B or n != min(self.B, self.n - win_begin):
            return None
        k = win_begin // self.B
        if not 0 <= k < len(self.brp) - 1:
            return None
        return self.brp[k], self.brp[k + 1] - self.brp[k]


def choose_route(algo, lazy, det, rec, win_begin, n, identity=False):
    """The launches (DESIGN.md §4.14) CbowModel.fwdbwd runs for windows [win_begin, win_begin + n) of a list whose
    _WindowList is ``rec`` (None: nothing prepared; ``identity``: the list is None, every window of the table).  A
    lazy or deterministic batch that was not planned raises RuntimeError: nothing falls back to the scatter."""
    def unplanned(mode):
        return RuntimeError("%s: windows [%d, %d) of this list were not given to prepare_batches"
                            % (mode, win_begin, win_begin + n))
    if lazy:
        if rec is None or rec.batch(win_begin, n) is None:
            raise unplanned("optimizer='lazy_adam'")
        return "batch_lazy"
    whole = rec is not None and rec.whole(win_begin, n)
    if algo == "rank1":
        return "r1_csc" if whole else "r1"
    if det:
        if whole:
            return "csc_det"
        if identity:
            raise RuntimeError("deterministic=True: fwdbwd needs a window list given to prepare_csc or prepare_batches")
        if rec is None or rec.batch(win_begin, n) is None:
            raise unplanned("deterministic=True")
        return "batch_det"
    if rec is not None and (win_begin, n) in rec.slabs:
        return "slabs"
    return "csc" if whole else "scatter"


def _nvl_setup(group, n_flat, dev):
    """Symmetric-memory buffers for the parameters and the gradient (torch.distributed._symmetric_memory: peer-mapped
    allocations + signal pads for cross-GPU barriers; NVLS multicast address when the NVSwitch fabric offers it).
    Returns None -- the caller then uses NCCL -- if G2V_CBOW_NVL=0 or the rendezvous is not possible on this box."""
    import os
    import sys
    if os.environ.get("G2V_CBOW_NVL", "1") == "0":
        return None
    try:
        import torch.distributed as dist
        import torch.distributed._symmetric_memory as symm
        w = symm.empty(n_flat, dtype=torch.float32, device=dev)
        g = symm.empty(n_flat, dtype=torch.float32, device=dev)
        hw, hg = symm.rendezvous(w, group), symm.rendezvous(g, group)
        mc = os.environ.get("G2V_CBOW_NVL_MULTICAST", "1") != "0"
        w_mc = int(hw.multicast_ptr or 0) if mc else 0       # 0: no NVLS multicast object behind this allocation
        g_mc = int(hg.multicast_ptr or 0) if mc else 0
        if not (w_mc and g_mc):
            w_mc = g_mc = 0
        return {"w": w, "g": g, "hw": hw, "hg": hg, "w_mc": w_mc, "g_mc": g_mc, "rank": dist.get_rank(group),
                "world": dist.get_world_size(group)}
    except Exception as exc:                   # no symmetric memory here: NCCL all-reduce + replicated update instead
        print("g2vec_b200: symmetric memory unavailable (%r); using NCCL for the gradient exchange" % (exc,), file=sys.stderr)
        return None


class _PlanBuffers:
    """Outputs and workspace of g2v_cbow_batch_plan for one window list of a CbowModel (n windows, batches of B),
    sized once from the list's incidence count, which no reordering of the list changes."""

    def __init__(self, model, win, B):
        self.m, self.n, self.B = model, int(win.shape[0]), int(B)
        w = win.to(torch.int64)
        self.nnz = int((model.rowptr[w + 1] - model.rowptr[w]).sum())
        dev, i32 = model.device, torch.int32
        self.n_b = -(-self.n // self.B)
        self.rows = torch.empty(max(self.nnz, 1), dtype=i32, device=dev)
        self.segptr = torch.empty(self.nnz + 1, dtype=i32, device=dev)
        self.pos = torch.empty(max(self.nnz, 1), dtype=i32, device=dev)
        self.brp = torch.empty(self.n_b + 1, dtype=i32, device=dev)
        nbytes = int(model.lib.g2v_cbow_batch_plan_workspace_bytes(self.n, self.nnz, self.B, model.V))
        self.ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)

    def build(self, win):
        """Build the plan of ``win`` (same length as the list this was sized for), then read the per-batch row offsets
        back (the only host synchronisation); returns (rows, segptr, pos) cut to their sizes and the row offsets as
        int64 NumPy [n_b + 1]."""
        m = self.m
        m._launch("g2v_cbow_batch_plan", m.rowptr.data_ptr(), m.gene.data_ptr(), win.data_ptr(), self.n, self.nnz,
                  self.B, m.V, self.rows.data_ptr(), self.segptr.data_ptr(), self.pos.data_ptr(), self.brp.data_ptr(),
                  self.ws.data_ptr())
        brp = self.brp.cpu().numpy().astype(np.int64)
        if brp[-1] < 0:
            raise RuntimeError("g2v_cbow_batch_plan: the list has more incidences than it was sized for")
        S = int(brp[-1])
        return self.rows[:S], self.segptr[:S + 1], self.pos[:self.nnz], brp


def batch_plan(model, win, batch):
    """The transposed incidence of every batch of ``batch`` consecutive windows of ``win`` (int32 device tensor), as
    device tensors (rows, segptr, pos, batch_rowptr) -- what prepare_batches records (g2v_cbow_batch_plan)."""
    n = int(win.shape[0])
    B = min(int(batch), n) if batch > 0 else n
    rows, segptr, pos, brp = _PlanBuffers(model, win, B).build(win)
    return rows, segptr, pos, torch.from_numpy(brp.astype(np.int32)).to(model.device)


def epoch_order(tr, seed, epoch, rank=0, world=1, out=None):
    """Rank ``rank``'s share of epoch ``epoch``'s list: out[i] = tr[P(rank + i*world)], P = P(seed, epoch, len(tr)) the
    pseudo-random permutation of DESIGN.md §4.12 (g2v_cbow_epoch_order).  ``tr``: int32 device tensor."""
    n = int(tr.shape[0])
    n_loc = max(0, -(-(n - rank) // world))
    if out is None:
        out = torch.empty(n_loc, dtype=torch.int32, device=tr.device)
    if out.shape[0] != n_loc or out.dtype != torch.int32:
        raise ValueError("epoch_order: out must be int32 [%d]" % n_loc)
    lib = _capi.load()
    _capi.check(lib.g2v_cbow_epoch_order(tr.data_ptr(), n, int(seed) & 0xFFFFFFFFFFFFFFFF, int(epoch), int(rank),
                                         int(world), out.data_ptr(),
                                         torch.cuda.current_stream(tr.device).cuda_stream), "g2v_cbow_epoch_order")
    return out


class WindowFeeder:
    """Feeds a CbowModel's context windows from pinned host memory, double-buffered.

    ``upload(k)`` enqueues, on a private copy stream, the host->device copies of the window CSR into buffer
    set k (gene ids travel as int16 when n_genes <= 32768 and are widened to int32 on the device: half the
    PCIe bytes); ``use(k)`` makes the compute stream wait for that upload and points the model at buffer set
    k; ``release(k)`` marks the set free once the step that read it has been enqueued."""

    def __init__(self, model, rowptr, gene, label):
        self.m = model
        dev = model.device
        to_np = lambda a: a.cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)
        rp, ge, la = to_np(rowptr).astype(np.int32), to_np(gene), to_np(label).astype(np.uint8)
        self.narrow = model.V <= 32768
        ge = ge.astype(np.int16 if self.narrow else np.int32)
        self.pins = [torch.from_numpy(np.ascontiguousarray(a)).pin_memory() for a in (rp, ge, la)]
        mk = lambda: [torch.empty(rp.shape[0], dtype=torch.int32, device=dev),
                      torch.empty(ge.shape[0], dtype=torch.int32, device=dev),
                      torch.empty(la.shape[0], dtype=torch.uint8, device=dev)]
        self.bufs = [mk(), mk()]
        self.stage = [torch.empty(ge.shape[0], dtype=torch.int16, device=dev) for _ in (0, 1)] if self.narrow else None
        self.stream = torch.cuda.Stream(device=dev)
        self.ready = [torch.cuda.Event(), torch.cuda.Event()]
        self.freed = [torch.cuda.Event(), torch.cuda.Event()]
        for k in (0, 1):
            self.freed[k].record(torch.cuda.current_stream(dev))
        self.h2d_bytes = int(sum(p.numel() * p.element_size() for p in self.pins))

    def upload(self, k):
        with torch.cuda.stream(self.stream):
            self.stream.wait_event(self.freed[k])            # the step that last read this set is done
            b = self.bufs[k]
            b[0].copy_(self.pins[0], non_blocking=True)
            if self.narrow:
                self.stage[k].copy_(self.pins[1], non_blocking=True)
                b[1].copy_(self.stage[k])                    # int16 -> int32 on the device
            else:
                b[1].copy_(self.pins[1], non_blocking=True)
            b[2].copy_(self.pins[2], non_blocking=True)
            self.ready[k].record(self.stream)

    def use(self, k):
        torch.cuda.current_stream(self.m.device).wait_event(self.ready[k])
        self.m.rowptr, self.m.gene, self.m.label = self.bufs[k]

    def release(self, k):
        self.freed[k].record(torch.cuda.current_stream(self.m.device))


def _dist():
    import torch.distributed as dist
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        return dist
    return None


def train_cbow(win_rowptr, win_gene, labels, n_genes, hidden, lr, max_epoch=500, seed=0, optimizer="adam",
               reduce="sum", W_ih0=None, W_ho0=None, split=None, early_stop=True, log=print, return_info=False,
               eval_train="lazy", algo="rows", batch=0, use_graph=True, reshuffle=False, deterministic=False,
               patience=1, lr_patience=0, lr_factor=0.1, min_lr=0.0, weight_decay=0.0, monitor="val_acc",
               class_weight=None):
    """Train the modified CBOW on CSR windows and return W_ih (np.float32 [n_genes, hidden]) exactly as
    ``compute_genetovec`` does: the weights after the last step whose validation accuracy did not drop.

    ``class_weight`` (None, the default, = off; "balanced"; or a pair (w0, w1) of finite numbers > 0): per-class
    weights of the training loss, Keras ``fit(class_weight=...)`` (DESIGN.md §4.20).  A window of label y counts with
    w_y: the step's cost is (1/N) sum_n w_{y_n} l_n over its N windows (not normalised by the weights), so
    dO = fl(fl(fl(sigmoid(o) - y) / N) * w_y), and the logged training loss is the weighted sum.  "balanced" is
    sklearn's: w_y = float32(n_tr / (2 n_tr,y)) from the labels of the whole training split (the same on every rank);
    a split without both labels is an error.  The accuracy counts, the validation loss and every early-stop and
    learning-rate decision keep their definitions.  w = (1, 1) gives the bits of an unweighted run.

    ``monitor``: what early stopping (``patience``) and the reduce-on-plateau rate (``lr_patience``) decide on.
    "val_acc" (the default): the correct validation count, the reference's rule.  "val_loss": the validation loss
    (DESIGN.md §4.19), the mean sigmoid BCE of the collapsed logits z = scale * sum_{g in n} (W_ih W_ho)[g] over the
    validation windows, each term capped at 64 and summed as the exact integer Q = sum rint(min(l, 64) 2^24) (the same
    for every launch grid and split over the ranks).  Both rules are the ones above with the count replaced by -Q: a
    step whose Q is <= the best so far becomes the best (ties: the later step) and the ``patience``-th step in a row
    with a higher Q stops the run; for the rate, only a Q below the best is an improvement.  The epoch lines then show
    ``LOSS[val]`` = Q 2^-24 / n_val after ``ACC[tr]``.

    ``weight_decay`` (λ, finite, 0 <= λ < 1 in float32; 0, the default, = off): decoupled weight decay, AdamW / SGDW
    as TF1's DecoupledWeightDecayExtension applies it (DESIGN.md §4.18).  Every optimizer step first sets each element
    it updates to fl(w - fl(λ w)), then takes the unchanged Adam / SGD step on that value with the gradient of the
    weights before the step.  adam, sgd and rank1 decay all of W_ih and W_ho every step; lazy_adam decays the rows its
    batch gathered, once each, and all of W_ho.  λ is a constant: the learning-rate schedule does not scale it, and
    the logged loss has no penalty term.

    ``lr_patience`` (int >= 0; 0, the default, = off): reduce the learning rate on a plateau, Keras
    ReduceLROnPlateau(mode="max", min_delta=0, cooldown=0) on the correct validation count of each step (DESIGN.md
    §4.17).  A count above the best so far is an improvement -- a tie is not, unlike the early-stop rule --; after
    ``lr_patience`` steps in a row without one the rate becomes max(float32(lr * ``lr_factor``), ``min_lr``) if it is
    above ``min_lr``, and the count starts again.  A step trains with the rate the decisions of the steps before it
    left.  The rule runs on the device, independent of early stopping, which still decides the stop and the returned
    weights.  Adam and lazy_adam only.

    ``patience`` (int >= 1, with ``early_stop``): the best validation count so far is tracked, a step whose count is
    >= the best becomes the best (ties: the later step), and the run stops at the ``patience``-th step in a row below
    the best (DESIGN.md §4.15).  The result is the best step's W_ih, also when the run ends at ``max_epoch``.  The
    default 1 is the reference's rule: stop at the first drop, return the weights from before it.

    ``max_epoch`` is the reference's ``--epoch`` (parsed at G2Vec.py:515 but ignored there; the loop is
    hard-coded ``range(500)`` at :262) -- the default 500 reproduces the reference.

    ``batch``: 0 (default) = full batch, one optimizer step per epoch over all training windows as the
    reference does (:262-264).  ``batch = B > 0`` is the north_star's mini-batch variant: the (already
    shuffled) training windows are cut into consecutive batches of B, one optimizer step (and, multi-GPU,
    one gradient all-reduce) per batch, loss mean over the batch; ``batch >= n_train`` equals full batch.

    ``use_graph``: on one GPU with full batch, every step after the first replays a CUDA graph of the step's
    launches (the Adam step size lives on the device, g2v_cbow_adam_tick), so the host only replays, waits
    and applies the early-stop rule.

    ``optimizer``: "adam" (TF1 AdamOptimizer, the reference's), "sgd", or "lazy_adam": TF1 LazyAdam on the
    embedding-lookup form of the model -- a step updates W_ih / m / v only on the rows of the genes its batch
    gathered (dense Adam on W_ho).  Full batch and without ``weight_decay`` it computes what "adam" computes (rows
    outside the training list keep zero gradient and zero moments; with decay "adam" shrinks them and lazy_adam does
    not); with ``batch`` it is the usual sparse mini-batch embedding update.
    Only with algo="rows", on one GPU.

    ``reshuffle`` (with 0 < ``batch`` < n_train): epoch 0 trains on the split's order, epoch e >= 1 on tr[P(seed, e)],
    P a pseudo-random permutation of the training list that depends on (seed, e, n_train) only (DESIGN.md §4.12), cut
    into consecutive batches as before; several GPUs deal the epoch's list as they deal the split's.  The order is
    written on the device every epoch, and lazy_adam rebuilds its batch plans there.  With ``batch >= n_train`` (full
    batch) the flag has no effect; with ``batch <= 0`` it is an error.

    ``deterministic`` (algo="rows", one GPU): every floating-point sum of a step is taken in a fixed order (DESIGN.md
    §4.13), so the same inputs and seed give the same bits of W_ih, W_ho, the history and the stop step on every run
    and for any launch grid -- every optimizer, full batch or mini-batches, with or without ``reshuffle`` and CUDA
    graphs, at every table size (no gene slabs).  Mini-batch adam/sgd then build per-batch plans as lazy_adam does.
    algo="rank1" is already reproducible with a full batch and is accepted unchanged; with ``batch > 0`` it is an error.

    ``return_info=True`` also returns a dict: ``history`` [(step, ACC[val], ACC[tr])], ``stop_step`` (the step where
    the run stopped early, else None), ``best_step`` (the step whose W_ih is returned; None if no step ran), ``lr``
    (the float32 learning rate each step trained with), ``lr_reductions`` (the steps whose decision cut the rate;
    one on the last step has no effect), ``val_loss`` (with monitor="val_loss": the mean validation loss of every step),
    ``class_weight`` (the float32 weights (w0, w1) the training loss used, None without), and more.
    """
    dist = _dist()
    check_config(algo, optimizer, deterministic, several_gpus=dist is not None, batch=batch, reshuffle=reshuffle,
                 patience=patience, lr_patience=lr_patience, lr_factor=lr_factor, min_lr=min_lr,
                 weight_decay=weight_decay, monitor=monitor, class_weight=class_weight)
    world, rank =(dist.get_world_size(), dist.get_rank()) if dist else (1, 0)
    rowptr_np = (win_rowptr.cpu().numpy() if isinstance(win_rowptr, torch.Tensor) else np.asarray(win_rowptr))
    N = rowptr_np.shape[0] - 1
    if N < 2:
        raise ValueError("need at least two context windows")
    tr, va = split_indices(N, seed) if split is None else split
    if isinstance(class_weight, str):            # "balanced", from the global training split
        class_weight = balanced_class_weight(labels, tr)
    if W_ih0 is None or W_ho0 is None:
        W_ih0, W_ho0 = init_weights(n_genes, hidden, seed)
    model = CbowModel(win_rowptr, win_gene, labels, n_genes, hidden, W_ih0, W_ho0, optimizer, reduce, lr, algo=algo,
                      nvl_group=dist.group.WORLD if (dist and algo == "rows") else None,
                      deterministic=deterministic and algo == "rows", weight_decay=weight_decay,
                      class_weight=class_weight)
    if lr_patience > 0:
        model.set_lr_plateau(lr_patience, lr_factor, min_lr, max_epoch)
    lens = np.diff(rowptr_np).astype(np.int64)
    n_tr, n_va = len(tr), len(va)
    full_batch = batch <= 0 or batch >= n_tr
    tr_loc = shard_by_nnz(np.asarray(tr), lens, world, rank, keep_order=not full_batch)
    va_loc = shard_by_nnz(np.asarray(va), lens, world, rank)
    dev = model.device
    tr_d = torch.from_numpy(np.ascontiguousarray(tr_loc, dtype=np.int32)).to(dev)
    reshuffle = bool(reshuffle) and not full_batch
    tr_all = None
    if reshuffle:                                # every rank deals each epoch's list from the global training list
        tr_all = tr_d if world == 1 else torch.from_numpy(np.ascontiguousarray(tr, dtype=np.int32)).to(dev)
    va_d = torch.from_numpy(np.ascontiguousarray(va_loc, dtype=np.int32)).to(dev)

    slabs = False
    if model.lazy or (model.det and not full_batch):   # touched genes of every batch; single-pass forward at every size
        model.prepare_batches(tr_d, len(tr_loc) if full_batch else batch)
    elif algo == "rows" and full_batch:          # tables larger than the L2: gene-slab passes over the static lists
        slabs = model.prepare_slabs(tr_d)
        model.prepare_slabs(va_d)
    if full_batch and len(tr_loc) and not slabs and not model.lazy:   # per-gene dO sums over the static training list
        model.prepare_csc(tr_d)
    if log:
        log("     Start training the modified CBOW with early stopping")
        if model.cw is not None:
            log("     class weights: w0=%.9g w1=%.9g" % model.cw)
    if max_epoch <= 0:                           # no optimizer step at all: the initial vectors
        out, hist, stop, best, plateau, info = model.W_ih, [], None, None, None, None
    elif full_batch:
        out, hist, stop, best, plateau, info = _device_loop(model, dist, tr_d, va_d, n_tr, n_va, len(tr_loc),
                                                            len(va_loc), max_epoch, early_stop, log, eval_train,
                                                            use_graph, patience=patience, monitor=monitor)
    else:
        out, hist, stop, best, plateau, info = _minibatch_loop(model, dist, world, tr_d, va_d, n_tr, n_va, len(tr_loc),
                                                               len(va_loc), max_epoch, early_stop, log, batch,
                                                               reshuffle=(tr_all, seed, rank) if reshuffle else None,
                                                               patience=patience, monitor=monitor)
    if log:
        log("    Optimization Finish")
    out = out.cpu().numpy()
    if return_info:
        rates, cuts = lr_rates(plateau) if plateau is not None else ([float(np.float32(lr))] * len(hist), [])
        res = {"history": hist, "stop_step": stop, "best_step": best, "n_train": n_tr, "n_val": n_va,
               "lr": rates, "lr_reductions": cuts, "model": model,
               "windows": (tr_d, va_d),
               "graph": bool(getattr(model, "loop_used_graph", False)), "exchange": model.exchange() if dist else None,
               "class_weight": model.cw}
        if monitor == "val_loss":
            res["val_loss"] = list(info.losses) if info is not None else []
        return out, res
    return out


def lr_rates(state):
    """From a host copy (int64 tensor) of a g2v_cbow_lr_plateau state: the float32 rate each decided step trained
    with, as floats, and the steps whose decision cut the rate."""
    n = int(state[4])
    f = state.numpy()[8:].view(np.float32)
    rates = f[4:4 + n]
    after = np.append(rates[1:], f[0])
    return [float(r) for r in rates], [s for s in range(n) if after[s] < rates[s]]


def lr_cut(state, step):
    """The rate the decision of ``step`` (already decided in the host copy ``state``) left if it cut the rate, else
    None."""
    n = int(state[4])
    f = state.numpy()[8:].view(np.float32)
    after = f[4 + step + 1] if step + 1 < n else f[0]
    return float(after) if after < f[4 + step] else None


class _LoopLog:
    """The host side of the reference loop body after the three session runs (G2Vec.py:268-283): log line every
    5th step, the Epoch(stop) line, the history.  Fed one step at a time with the step's counters.

    It also follows the early-stop rule with ``patience`` (DESIGN.md §4.15) on the integer validation counts, as
    g2v_cbow_loop_decide[_best] do: ``best_step`` is the step whose weights the loop returns.  ``patience=None``: no
    early stopping, every step is the new best (the loop returns the last weights).

    ``monitor="val_loss"`` (DESIGN.md §4.19): the rule decides on the score 2^62 - Q of the step's validation loss Q
    (passed as ``q``) instead of the count, as g2v_cbow_loop_decide[_best]_score do, and every epoch line shows the mean
    loss as ``LOSS[val]`` after ``ACC[tr]``; ``losses`` holds it for every step."""

    def __init__(self, n_tr, n_va, log, patience=1, monitor="val_acc"):
        self.n_tr, self.n_va, self.log = n_tr, n_va, log
        self.hist, self.t0 = [], time.time()
        self.patience = patience
        self.best_val, self.best_step, self.bad = -1, None, 0
        # reduce-on-plateau: a host copy of the rate state whose decisions step() reports (set by the loop), else None
        self.plateau = None
        self.loss = monitor == "val_loss"
        self.losses = []

    def _value(self, acc, q):
        return SCORE_TOP - int(q) if self.loss else int(acc[2])

    def _loss_txt(self, step):
        return "\tLOSS[val]=%.6f" % self.losses[step] if self.loss else ""

    def stops(self, acc, q=0):
        """Whether a step with counters ``acc`` (and validation loss ``q``) ends the run under the rule (host-driven
        loops decide with this)."""
        return self.patience is not None and self._value(acc, q) < self.best_val and self.bad + 1 >= self.patience

    def step(self, step, acc, shown, stopped_here, q=0):
        f32 = np.float32
        acc_val = f32(int(acc[2])) / f32(max(self.n_va, 1))
        acc_tr_prev = f32(int(acc[1])) / f32(max(self.n_tr, 1))      # = ACC[tr] of step-1 (SURVEY 3.2-5)
        acc_tr = f32(int(acc[3])) / f32(max(self.n_tr, 1)) if shown else None
        hist, log = self.hist, self.log
        if hist and hist[-1][2] is None:
            hist[-1] = (hist[-1][0], hist[-1][1], float(acc_tr_prev))
        hist.append((step, float(acc_val), None if acc_tr is None else float(acc_tr)))
        if self.loss:
            self.losses.append(val_loss_mean(q, self.n_va))
        v = self._value(acc, q)
        if self.patience is None or v >= self.best_val:
            self.best_val, self.best_step, self.bad = v, step, 0
        else:
            self.bad += 1
        if step % 5 == 0 and log:
            t1 = time.time()
            log("    - Epoch: %03d\tACC[val]=%.4f\tACC[tr]=%.4f%s (%.3f sec)" % (step, acc_val, acc_tr,
                                                                          self._loss_txt(step), t1 - self.t0))
            self.t0 = time.time()
        if self.plateau is not None and log:
            cut = lr_cut(self.plateau, step)
            if cut is not None:
                log("    - Epoch: %03d\tlearning rate -> %g" % (step, cut))
        if stopped_here:
            # the best step's accuracies; its ACC[tr] is in the history by now (step-1's was filled in above)
            if log:
                b = hist[self.best_step]
                log("    - Epoch(stop): %03d\tACC[val]=%.4f\tACC[tr]=%.4f%s (%.3f sec)"
                    % (b[0], b[1], b[2], self._loss_txt(b[0]), time.time() - self.t0))
            return True
        return False

    def end(self):
        """After a run that reached max_epoch: the Epoch(best) line if the best step is not the last one, which only
        patience > 1 allows.  Call it once the last step's ACC[tr] is in the history."""
        if self.log and self.hist and self.best_step != self.hist[-1][0]:
            b = self.hist[self.best_step]
            self.log("    - Epoch(best): %03d\tACC[val]=%.4f\tACC[tr]=%.4f" % b + self._loss_txt(b[0]))


class DeviceLoop:
    """One model's training loop state on the device (g2v_cbow_loop_*) and the launches of one iteration of the
    reference loop (G2Vec.py:262-267): snapshot + zero counters, fwd+bwd, [all-reduce], optimizer, validation
    accuracy, [training accuracy], [all-reduce of the counters], decide.  Used by train_cbow and by bench.py.

    Carried mode (``self.carried``: one GPU, rows, dense optimizer, fwdbwd on the CSC path of the training list):
    the training-accuracy pass runs on every step as the tail pass (g2v_cbow_loop_tail) and is also the next step's
    forward, so the next fwdbwd only expands its dO into g_ih.  On the csc path with the certified validation pass
    (monitor="val_acc", D in TAIL_VAL_D) the validation pass runs inside the tail's launch (g2v_cbow_loop_tail_val).  The training list is gathered once per step instead
    of twice.  This assumes the training windows do not change between steps: the list is static, and a
    WindowFeeder re-uploads the same windows every step.  The first step after reset() runs the full forward,
    decided on the device, so a graph captured right after reset() is correct from its first replay.

    Patience (``early_stop`` with ``patience`` > 1, DESIGN.md §4.15): no snapshot at the start of a step; the decision
    is g2v_cbow_loop_decide_best, followed by g2v_cbow_loop_keep_best, which copies W_ih into ``result`` on the steps
    that improve on the best validation count.  ``result`` then holds the best step's weights however the loop ends.

    ``monitor="val_loss"`` (DESIGN.md §4.19): the validation pass also computes the loss Q, and both rules decide on the
    score 2^62 - Q (g2v_cbow_loop_decide[_best]_score), recorded per step in ``score_d`` (host copy ``score_pin``)."""

    # the smallest patience that takes the keep-best kernels; tests lower it to 1 to check them against the default rule
    keep_best_from = 2

    def __init__(self, model, dist, tr_d, va_d, n_tr, max_epoch, early_stop, snapshot=True, patience=1,
                 monitor="val_acc"):
        self.m, self.dist, self.tr_d, self.va_d, self.n_tr = model, dist, tr_d, va_d, n_tr
        self.n_tr_loc, self.n_va_loc = int(tr_d.shape[0]), int(va_d.shape[0])
        self.carried = (dist is None and not model.lazy and self.n_tr_loc > 0
                        and model.route(tr_d) in ("csc", "csc_det"))
        self.loss = monitor == "val_loss"
        dev = model.device
        self.ctl = torch.zeros(8, dtype=torch.int64, device=dev)
        n_hist = max(max_epoch, 1) * 4
        # val_loss: one score per step, after the counters in the same allocation (symmetric memory with NVLink)
        n_score = max(max_epoch, 1) if self.loss else 0
        # with the NVLink exchange the history lives in symmetric memory and the accuracy counters of all ranks are
        # added into it by the ranks themselves (g2v_cbow_loop_counters_nvl): no NCCL call is left in the step
        self.hist_nvl = None
        if dist and model.nvl:
            try:
                import torch.distributed._symmetric_memory as symm
                h = symm.empty(n_hist + n_score, dtype=torch.int64, device=dev)
                hh = symm.rendezvous(h, dist.group.WORLD)
                self.hist_nvl = {"h": hh, "mc": int(hh.multicast_ptr or 0) if model.nvl["g_mc"] else 0}
                self.hist_all = h
            except Exception:
                self.hist_nvl = None
        if self.hist_nvl is None:
            self.hist_all = torch.zeros(n_hist + n_score, dtype=torch.int64, device=dev)
        self.hist_d, self.score_d = self.hist_all[:n_hist], self.hist_all[n_hist:]
        self.score_pin = torch.zeros(n_score, dtype=torch.int64).pin_memory() if self.loss else None
        self.ctl_pin = torch.zeros(8, dtype=torch.int64).pin_memory()
        self.hist_pin = torch.zeros(max(max_epoch, 1) * 4, dtype=torch.int64).pin_memory()
        self.max_epoch, self.early_stop, self.patience = int(max_epoch), bool(early_stop), int(patience)
        # best: {patience, best_step, bad_steps, improved} of the keep-best path, else None
        self.best = self.best_pin = None
        if self.early_stop and self.patience >= self.keep_best_from:
            self.best = torch.zeros(4, dtype=torch.int64, device=dev)
            self.best_pin = torch.zeros(4, dtype=torch.int64).pin_memory()
        # default path: W_ih before the step being decided (only an early stop ever returns it); keep-best path: W_ih
        # of the best step so far
        self.result = model.W_ih.clone() if (snapshot or self.best is not None) else None
        # the model's reduce-on-plateau state, read back with the loop's status (model.set_lr_plateau, else None)
        self.plateau_pin = torch.empty_like(model.plateau, device="cpu").pin_memory() if model.plateau is not None \
            else None
        self.reset()

    def reset(self):
        self.m._launch("g2v_cbow_loop_init", self.ctl.data_ptr(), self.max_epoch, int(self.early_stop))
        self.m.lr_reset()
        if self.best is not None:
            self.best.copy_(torch.tensor([self.patience, -1, 0, 0], dtype=torch.int64))
        if self.carried:                             # drop a pending carry: its g_ho partial would be added twice
            self.m.g_ho.zero_()
            self.m.acc[4:].zero_()
        if self.loss:                                # each decision clears Q; drop one a caller left pending
            self.m.q.zero_()
        if self.hist_nvl:
            self.hist_nvl["h"].barrier(channel=2)    # no rank is still adding into the history of the previous loop
            self.hist_all.zero_()
            self.hist_nvl["h"].barrier(channel=2)    # ... and no rank adds before every history is zero

    def attach(self):
        _capi.check(self.m.lib.g2v_cbow_loop_attach(self.ctl.data_ptr()), "g2v_cbow_loop_attach")

    def detach(self):
        _capi.check(self.m.lib.g2v_cbow_loop_attach(None), "g2v_cbow_loop_attach")

    def one(self, show, m_fb=None, m_upd=None, m_val=None):
        """Enqueue one iteration (the optional events mark the end of fwd+bwd, of the update, of the validation pass).
        In carried mode ``show`` changes nothing: ACC[tr] comes from the tail pass on every step."""
        m, dist = self.m, self.dist
        m._launch("g2v_cbow_loop_begin", self.ctl.data_ptr(), m.acc.data_ptr(), m.W_ih.data_ptr(),
                  None if (self.result is None or self.best is not None) else self.result.data_ptr(), m.V * m.D)
        if self.n_tr_loc:
            m.fwdbwd(self.tr_d, self.n_tr)       # acc[1] += correct predictions with the PRE-update weights
                                                 # (carried: the forward is skipped on the device, acc[1] carried)
        if m_fb is not None:
            m_fb.record()
        if dist:
            for g in m.grad_tensors():
                dist.all_reduce(g)               # rows: ONE collective over [g_ih | g_ho]; rank1: c
        m.update()
        if m_upd is not None:
            m_upd.record()
        # the carried csc step with the certified validation pass runs both window passes in one launch (§4.32)
        tail_val = (self.carried and not m.det and not self.loss and self.n_va_loc and m.D in TAIL_VAL_D
                    and choose_route(m.algo, False, False, m.prepared(self.va_d), 0, self.n_va_loc) in ("csc", "scatter"))
        if self.n_va_loc and not tail_val:
            if self.loss:
                m.evaluate(self.va_d, 2, loss=True)
            else:
                m.evaluate(self.va_d, 2)
        if m_val is not None:
            m_val.record()
        if tail_val:
            m.loop_tail_val(self.ctl, self.tr_d, self.n_tr, self.va_d)
        elif self.carried:
            m.loop_tail(self.ctl, self.tr_d, self.n_tr)
        elif show and self.n_tr_loc:
            m.evaluate(self.tr_d, 3)
        acc_ptr = m.acc.data_ptr()
        q_ptr = m.q.data_ptr() if self.loss else None
        if self.hist_nvl:
            hn = self.hist_nvl
            m._launch("g2v_cbow_loop_counters_nvl", self.ctl.data_ptr(), acc_ptr, hn["h"].buffer_ptrs_dev, hn["mc"],
                      m.nvl["world"])
            if self.loss:                            # Q of every rank into score[step] of every rank
                m._launch("g2v_cbow_loop_score_nvl", self.ctl.data_ptr(), q_ptr, hn["h"].buffer_ptrs_dev, hn["mc"],
                          self.hist_d.numel(), m.nvl["world"])
            hn["h"].barrier(channel=3)
            acc_ptr = q_ptr = None                   # decide on the sums already in hist[step] (and score[step])
        elif dist:
            dist.all_reduce(m.acc[1:4])
            if self.loss:
                dist.all_reduce(m.q)
        if self.best is None:
            if self.loss:
                m._launch("g2v_cbow_loop_decide_score", self.ctl.data_ptr(), acc_ptr, self.hist_d.data_ptr(), q_ptr,
                          self.score_d.data_ptr())
            else:
                m._launch("g2v_cbow_loop_decide", self.ctl.data_ptr(), acc_ptr, self.hist_d.data_ptr())
        else:
            if self.loss:
                m._launch("g2v_cbow_loop_decide_best_score", self.ctl.data_ptr(), self.best.data_ptr(), acc_ptr,
                          self.hist_d.data_ptr(), q_ptr, self.score_d.data_ptr())
            else:
                m._launch("g2v_cbow_loop_decide_best", self.ctl.data_ptr(), self.best.data_ptr(), acc_ptr,
                          self.hist_d.data_ptr())
            m._launch("g2v_cbow_loop_keep_best", self.best.data_ptr(), m.W_ih.data_ptr(), self.result.data_ptr(),
                      m.V * m.D)
        if m.plateau is not None:                # the rate rule on the value the decision just recorded
            if self.loss:
                m.lr_decide(self.score_d.data_ptr(), 1, self.ctl.data_ptr() + 8)
            else:
                m.lr_decide(self.hist_d.data_ptr() + 16, 4, self.ctl.data_ptr() + 8)

    def fetch(self):
        self.ctl_pin.copy_(self.ctl, non_blocking=True)
        self.hist_pin.copy_(self.hist_d, non_blocking=True)
        if self.score_pin is not None:
            self.score_pin.copy_(self.score_d, non_blocking=True)
        if self.best is not None:
            self.best_pin.copy_(self.best, non_blocking=True)
        if self.plateau_pin is not None:
            self.plateau_pin.copy_(self.m.plateau, non_blocking=True)

    def capture(self, pattern):
        """The iterations of `pattern` (list of show flags) + the status read-back as one CUDA graph."""
        g = torch.cuda.CUDAGraph()
        t_before = self.m.t
        with torch.cuda.graph(g):
            for sh in pattern:
                self.one(sh)
            self.fetch()
        self.m.t = t_before                      # capture records, it does not execute
        return g


def _device_loop(model, dist, tr_d, va_d, n_tr, n_va, n_tr_loc, n_va_loc, max_epoch, early_stop, log, eval_train,
                 use_graph, chunk=5, patience=1, monitor="val_acc"):
    """Full-batch loop of G2Vec.py:262-283 with the early-stop rule, the result snapshot and the step counter on
    the DEVICE (g2v_cbow_loop_*): the host enqueues `chunk` iterations at a time -- one CUDA-graph replay of
    4 plain iterations + 1 that also runs the training-accuracy pass (in carried mode, five identical iterations
    that all have it) -- and synchronises once per printed line instead of once per step.  Iterations enqueued after
    the stop are no-ops (every kernel tests ctl.stopped).  Multi-GPU: the all-reduces are part of the captured graph
    (NCCL is capturable); if capture is refused the same launches run eagerly.  Returns (W_ih to return, history,
    stop step or None, best step, host copy of the model's reduce-on-plateau state or None, the _LoopLog)."""
    dev = model.device
    loop = DeviceLoop(model, dist, tr_d, va_d, n_tr, max_epoch, early_stop, snapshot=bool(early_stop),
                      patience=patience, monitor=monitor)
    shown = lambda s: loop.carried or s % 5 == 0 or eval_train == "always"
    info = _LoopLog(n_tr, n_va, log, patience if early_stop else None, monitor=monitor)
    info.plateau = loop.plateau_pin

    def consume(lo, hi):
        """Host view of steps lo..hi-1 after a sync; True when the loop is over."""
        decided, stop_step = int(loop.ctl_pin[1]), int(loop.ctl_pin[2])
        for s in range(lo, min(hi, decided)):
            q = SCORE_TOP - int(loop.score_pin[s]) if loop.loss else 0
            if info.step(s, loop.hist_pin[4 * s:4 * s + 4], shown(s), s == stop_step, q):
                return True
        return bool(int(loop.ctl_pin[0]))

    loop.attach()
    graph = None
    try:
        loop.one(True); loop.fetch()             # step 0 eagerly: it also warms every kernel up before a capture
        torch.cuda.current_stream(dev).synchronize()
        done, over = 1, consume(0, 1)
        graph_failed, graph_pattern = not use_graph, None
        while not over and done < max_epoch:
            k = min(chunk, max_epoch - done)
            pattern = [shown(done + i) for i in range(k)]
            if k == chunk and not graph_failed and graph is None:
                try:
                    graph, graph_pattern = loop.capture(pattern), pattern
                except Exception:
                    if dist is None:
                        raise
                    graph_failed = True          # collectives not capturable here: same launches, eagerly
            if graph is not None and pattern == graph_pattern:
                model.t += k
                graph.replay()
            else:
                for sh in pattern:
                    loop.one(sh)
                loop.fetch()
            torch.cuda.current_stream(dev).synchronize()        # one host sync per `chunk` steps
            over = consume(done, done + k)
            done += k
        stop = int(loop.ctl_pin[2]) if int(loop.ctl_pin[2]) >= 0 else None
        if stop is None and info.hist and info.hist[-1][2] is None:
            # ACC[tr] of the last step was never needed for a log line; evaluate it once for the history (a carried
            # loop has it for every step)
            loop.detach()
            model.acc.zero_()
            if n_tr_loc:
                model.evaluate(tr_d, 3)
            if dist:
                dist.all_reduce(model.acc[1:4])
            a = model.acc.cpu()
            last = info.hist[-1]
            info.hist[-1] = (last[0], last[1], float(np.float32(int(a[3])) / np.float32(max(n_tr, 1))))
        if stop is None:
            info.end()
    finally:
        loop.detach()
    model.loop_used_graph = graph is not None
    if loop.best is not None:                    # keep-best path: result holds the best step's weights in every case
        return loop.result, info.hist, stop, int(loop.best_pin[1]), info.plateau, info
    # stopped early: the snapshot taken before the dropping step (G2Vec.py:283,286); else the final weights
    return (loop.result if stop is not None else model.W_ih), info.hist, stop, info.best_step, info.plateau, info


def _minibatch_loop(model, dist, world, tr_d, va_d, n_tr, n_va, n_tr_loc, n_va_loc, max_epoch, early_stop, log, batch,
                    reshuffle=None, patience=1, monitor="val_acc"):
    """north_star's mini-batch variant: one optimizer step (and one gradient all-reduce) per batch of the shuffled
    training list, the reference's per-epoch accuracies and early stop around it; host-driven, one sync per epoch.
    ``reshuffle`` = (global training list on the device, seed, rank): every epoch e >= 1 trains on this rank's share of
    the epoch's order, written into one preallocated buffer (g2v_cbow_epoch_order); lazy_adam then rebuilds the
    buffer's batch plans (one more sync), as does the deterministic mode.  The early-stop rule with ``patience`` is
    applied on the host after the epoch's sync; the result is copied on the epochs that improve on the best.  The
    reduce-on-plateau rule, if the model has it, is decided on the device after the counters' all-reduce and its state
    read back with them.  ``monitor="val_loss"``: the validation pass also adds the loss Q into model.q (all-reduced
    right after the counters), both rules decide on the score 2^62 - Q, and the rate rule reads the score on the device.
    Returns what _device_loop returns."""
    dev = model.device
    info = _LoopLog(n_tr, n_va, log, patience if early_stop else None, monitor=monitor)
    loss = monitor == "val_loss"
    score_d = torch.zeros(1, dtype=torch.int64, device=dev) if loss else None
    if model.plateau is not None:                # read back with each epoch's counters, for the log and the result
        model.lr_reset()
        info.plateau = torch.empty_like(model.plateau, device="cpu").pin_memory()
    result = model.W_ih.clone()
    stop = None
    per = -(-batch // world)
    ep_d = torch.empty_like(tr_d) if reshuffle else None
    for step in range(max_epoch):
        win = tr_d
        if reshuffle and step >= 1:
            tr_all, seed, rank = reshuffle
            epoch_order(tr_all, seed, step, rank, world, out=ep_d)
            if model.lazy or model.det:
                model.prepare_batches(ep_d, batch)
            win = ep_d
        model.acc.zero_()
        if loss:
            model.q.zero_()
        for lo in range(0, -(-n_tr // world), per):             # same trip count on every rank (collectives inside)
            nb = max(0, min(per, n_tr_loc - lo))
            nb_tot = nb
            if dist:
                t_nb = torch.tensor([nb], dtype=torch.int64, device=dev); dist.all_reduce(t_nb)
                nb_tot = int(t_nb[0])
            model.fwdbwd(win, nb_tot, win_begin=lo, n_win=nb)
            if dist:
                for g in model.grad_tensors():
                    dist.all_reduce(g)
            model.update()
        if n_va_loc:
            if loss:
                model.evaluate(va_d, 2, loss=True)
            else:
                model.evaluate(va_d, 2)
        if n_tr_loc:
            model.evaluate(tr_d, 3)                              # acc[1] mixes weights across batches: always evaluate
        if dist:
            dist.all_reduce(model.acc[1:4])
            if loss:
                dist.all_reduce(model.q)
        if loss:                                                 # score = 2^62 - Q, for the rate rule on the device
            torch.neg(model.q, out=score_d).add_(SCORE_TOP)
        if model.plateau is not None:                            # the rate rule on the epoch's (summed) count or score
            model.lr_decide(score_d.data_ptr() if loss else model.acc.data_ptr() + 16)
            info.plateau.copy_(model.plateau, non_blocking=True)
        acc = model.acc.cpu()                                    # the epoch's only host sync
        q = int(model.q.cpu()[0]) if loss else 0
        if info.step(step, acc, True, info.stops(acc, q), q):
            stop = step
            break
        if info.best_step == step:
            result.copy_(model.W_ih)
    if stop is None:
        info.end()
    return result, info.hist, stop, info.best_step, info.plateau, info


def compute_genetovec(pathList, n_genes, hidden_size, learning_rate, max_epoch=500, seed=0, log=print):
    """Drop-in for the reference signature (G2Vec.py:217): dense ``pathList`` [N, n_genes+1] in
    (last column = label), W_ih out."""
    from .paths import dense_pathlist_to_csr
    rowptr, gene, label = dense_pathlist_to_csr(pathList)
    return train_cbow(rowptr, gene, label, n_genes, hidden_size, learning_rate, max_epoch=max_epoch, seed=seed,
                      log=log)


def cbow_step_host(rowptr, gene, label, W_ih, W_ho, state=None, lr=0.005, t=1, optimizer="adam", reduce="sum",
                   beta1=0.9, beta2=0.999, eps=1e-8):
    """One full-batch step through ``g2v_cbow_step_host``: NumPy in, NumPy updated in place."""
    lib = _capi.load()
    rowptr = np.ascontiguousarray(rowptr, dtype=np.int32); gene = np.ascontiguousarray(gene, dtype=np.int32)
    label = np.ascontiguousarray(label, dtype=np.uint8)
    V, D = W_ih.shape
    for a in (W_ih, W_ho):
        assert a.dtype == np.float32 and a.flags.c_contiguous
    opt = {"adam": _capi.OPT_ADAM_TF1, "sgd": _capi.OPT_SGD}[optimizer]
    if opt == _capi.OPT_ADAM_TF1 and state is None:
        state = [np.zeros_like(W_ih), np.zeros_like(W_ih), np.zeros_like(W_ho), np.zeros_like(W_ho)]
    p = lambda a: 0 if a is None else a.ctypes.data
    m_ih, v_ih, m_ho, v_ho = state if state is not None else (None,) * 4
    loss = np.zeros(1, dtype=np.float64); nc = np.zeros(1, dtype=np.int64)
    rc = lib.g2v_cbow_step_host(rowptr.ctypes.data, gene.ctypes.data, label.ctypes.data, rowptr.shape[0] - 1,
                                gene.shape[0], W_ih.ctypes.data, W_ho.ctypes.data, p(m_ih), p(v_ih), p(m_ho),
                                p(v_ho), V, D, opt, {"sum": 0, "mean": 1}[reduce], lr, beta1, beta2, eps, t,
                                loss.ctypes.data, nc.ctypes.data)
    _capi.check(rc, "g2v_cbow_step_host")
    return state, float(loss[0]), int(nc[0])
