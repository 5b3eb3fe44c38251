"""The launch dispatch of the class-weighted and weight-decayed CBOW kernels, restated in Python, and a check that the
shape lists of tests/test_gpu_cbow_f64_options.py reach every (instantiation, branch) pair of it (no GPU needed).

Restated from g2vec_b200/csrc (the source checks below pin the expressions this restates):
  launch_rows       D in {128, 256, 512}: cbow_rows_kernel<VEC = D / 128>; any other D: cbow_rows_generic_kernel with
                    8 warps x 2 rows of D floats of dynamic shared memory (the opt-in attribute matters above 48 KB),
                    admitted while that plus its 16-byte static CtaAcc fits the opt-in limit;
  launch_rows_det   the same VEC split; cbow_rows_generic_det_kernel admitted while its dynamic part plus 1 KB fits;
  launch_r1_update  r1_update_kernel<VEC = D / 128> for D in {128, 256, 512}, else VEC = 0; 8 rows of D floats of
                    dynamic shared memory, the opt-in attribute set above 48 KB (D > 1536);
  cbow_update_kernel  float4 over V*D / 4 elements, then a scalar tail of V*D % 4 elements of W_ih and all of W_ho;
  g2v_cbow_lazy_adam_wd  the rows kernel's float4 path when D % 4 == 0, its scalar one otherwise; the W_ho step on
                    (D + 255) / 256 blocks of 256 threads.
The GPU file loops over both optimizers (Adam and SGD) inside each rank-1 and dense case."""
import os
import re

from tests import test_gpu_cbow_f64_options as opt

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "g2vec_b200", "csrc")
# cudaDevAttrMaxSharedMemoryPerBlockOptin of an H100 (227 KB); the largest D below follows from it
H100_OPTIN = 232448
DEFAULT_SMEM = 48 * 1024
WARPS = 8
ROWS_STATIC = 16           # sizeof(CtaAcc), the generic rows kernel's static shared memory
DET_RESERVE = 1024         # what launch_rows_det reserves for the generic deterministic kernel's static shared memory
VEC_D = {128: 1, 256: 2, 512: 4}


def _d(D):
    return opt.generic_max_d(H100_OPTIN) if D == "max" else D


def rows_branch(D, det=False):
    """(instantiation, branch) that launch_rows (det: launch_rows_det) takes at hidden size D."""
    if D in VEC_D:
        return ("vec%d" % VEC_D[D], "")
    smem = WARPS * 2 * D * 4
    if smem + (DET_RESERVE if det else ROWS_STATIC) > H100_OPTIN:
        return ("generic", "refused")
    return ("generic", ("opt-in" if smem > DEFAULT_SMEM else "48 KB") + (" D%4==0" if D % 4 == 0 else " D%4!=0"))


def r1_branch(D):
    smem = WARPS * D * 4
    if smem > H100_OPTIN:
        return ("vec%d" % VEC_D.get(D, 0), "refused")
    return ("vec%d" % VEC_D.get(D, 0), "opt-in" if smem > DEFAULT_SMEM else "48 KB")


def update_tail(V, D):
    return (V * D) % 4


def lazy_branch(D):
    return ("float4" if D % 4 == 0 else "scalar", "one W_ho block" if (D + 255) // 256 == 1 else "several W_ho blocks")


ROWS_PAIRS = {("vec1", ""), ("vec2", ""), ("vec4", "")} | {("generic", s + t) for s in ("48 KB", "opt-in")
                                                            for t in (" D%4==0", " D%4!=0")}


def test_the_restated_dispatch_is_the_source():
    src = open(os.path.join(CSRC, "g2v_cbow.cu")).read()
    r1 = open(os.path.join(CSRC, "g2v_cbow_rank1.cu")).read()
    flat = lambda s: re.sub(r"\s+", " ", s)
    src, r1 = flat(src), flat(r1)
    assert src.count("const size_t smem = (size_t)kCbowWarps * 2 * D * sizeof(float);") == 2
    assert "smem + fa.sharedSizeBytes <= (size_t)dp.max_smem_optin" in src
    assert "smem + 1024 <= (size_t)dp.max_smem_optin" in src
    assert src.count("if (D == 128) G2V_LAUNCH_VEC(1) else if (D == 256) G2V_LAUNCH_VEC(2) "
                     "else if (D == 512) G2V_LAUNCH_VEC(4)") == 1
    assert "if (D == 128) G2V_LAUNCH_DET(1) else if (D == 256) G2V_LAUNCH_DET(2) else if (D == 512) G2V_LAUNCH_DET(4)" \
        in src
    assert "cudaFuncSetAttribute(cbow_rows_generic_kernel<BACKWARD, CW>," in src
    assert "cudaFuncSetAttribute(cbow_rows_generic_det_kernel<CW>," in src
    common = flat(open(os.path.join(CSRC, "g2v_cbow_common.cuh")).read())
    assert ("struct CtaAcc { // per-CTA accumulators in shared memory double loss; unsigned long long correct; };"
            in common)
    assert "constexpr int kCbowWarps = %d;" % WARPS in common
    assert "const size_t smem = (size_t)kCbowWarps * D * sizeof(float);" in r1
    assert "if (smem > 48 * 1024) G2V_CUDA_OK(cudaFuncSetAttribute(r1_update_kernel<VEC, OPT, WD>," in r1
    assert "if (D == 128) rc = launch_r1_update<1, OPT, WD>" in r1
    assert "else if (D == 256) rc = launch_r1_update<2, OPT, WD>" in r1
    assert "else if (D == 512) rc = launch_r1_update<4, OPT, WD>" in r1
    assert "else rc = launch_r1_update<0, OPT, WD>" in r1
    assert "ho<<<(unsigned)((D + 255) / 256), 256, 0, st>>>" in src
    assert "for (int64_t i = (n4 << 2) + tid; i < n + n2; i += nthreads)" in src


def test_the_restated_limits():
    assert opt.generic_max_d(H100_OPTIN) == 3631 and opt.det_max_d(H100_OPTIN) == 3616
    assert rows_branch(3631) != ("generic", "refused") and rows_branch(3632) == ("generic", "refused")
    assert rows_branch(3616, det=True) != ("generic", "refused")
    assert rows_branch(3617, det=True) == ("generic", "refused")
    assert rows_branch(768)[1].startswith("48 KB") and rows_branch(769)[1].startswith("opt-in")
    assert r1_branch(1536) == ("vec0", "48 KB") and r1_branch(1537) == ("vec0", "opt-in")
    assert r1_branch(3631)[1] == "opt-in"


def test_class_weight_shapes_reach_every_rows_branch():
    Ds = [_d(D) for D, _, _ in opt.CW_CASES]
    assert {rows_branch(D) for D in Ds} == ROWS_PAIRS
    assert {rows_branch(D, det=True) for D in Ds} == ROWS_PAIRS | {("generic", "refused")}
    assert opt.generic_max_d(H100_OPTIN) in Ds                  # the largest D the weighted generic kernel admits
    assert any(V >= 4097 and D == "max" for D, V, _ in opt.CW_CASES)   # with 4096-gene windows
    # every weighted route but the gene slabs, both weights, every mode
    assert set(opt.CW_ROUTES) == {"fwdbwd", "fwdbwd_csc", "fwd_do", "fwdbwd_csc_det", "fwd_do_det", "loop_tail",
                                  "loop_tail_det", "r1_windows", "r1_windows_csc"}
    assert set(opt.DET_ROUTES) <= set(opt.CW_ROUTES)
    assert set(opt.MODES) == {(m, r) for m in ("dyadic", "realistic") for r in ("sum", "mean")}


def test_dense_decay_shapes_reach_every_tail():
    assert {update_tail(V, D) for D, V in opt.DENSE_WD_SHAPES} == {0, 1, 2, 3}
    assert {o for _, o in opt.DENSE_VARIANTS} == {opt.ADAM, opt.SGD}
    assert {n for n, _ in opt.DENSE_VARIANTS} == {"adam_host", "adam_dev", "sgd"}
    assert 1 in opt.DENSE_T and max(opt.DENSE_T) >= 1000 and len(opt.DENSE_LAMS) >= 2


def test_lazy_decay_shapes_reach_every_branch():
    got = {lazy_branch(_d(D)) for D, _, _ in opt.CW_CASES}
    assert got == {(a, b) for a in ("float4", "scalar") for b in ("one W_ho block", "several W_ho blocks")}


def test_rank1_decay_shapes_reach_every_branch():
    Ds = [_d(D) for D in opt.R1_DS]
    assert {r1_branch(D) for D in Ds} == {("vec1", "48 KB"), ("vec2", "48 KB"), ("vec4", "48 KB"), ("vec0", "48 KB"),
                                          ("vec0", "opt-in")}
    assert 1536 in Ds and 1537 in Ds and opt.generic_max_d(H100_OPTIN) in Ds     # both sides of the opt-in, largest D
    assert {D % 4 == 0 for D in Ds if D not in VEC_D} == {True, False}
    assert set(opt.R1_OPTS) == {opt.ADAM, opt.SGD}
