"""The training-stage kernels' formulas (csrc/bx_train.cu) against float64 without a GPU: the fp32 oracle of
oracle/train_stages.py (bit-identical to the kernels for the matches and, to the last ulp of sin / cos, for the
augmentation) held to the float64 restatements of the same file, which evaluate the reference's formulas
(get_matching_indices, kornia's axis_angle_to_rotation_matrix, EquiMatch, cal_so2_gt) and not the fp32 operation order.
tests/test_train_fp64_gpu.py holds the kernels to the same checks (oracle/train_cases.py).

The bounds (u = 2^-24; K constants in oracle/train_cases.py):

* Ground-truth matches.  q_j = ((R_j0 x + R_j1 y) + R_j2 z) + t_j in fp32 is four roundings of terms below
  sum_k |R_jk| |p_k| + |t_j|: |fl(q_j) - q_j| <= e_q,j = KQ u (sum_k |R_jk| |p_k| + |t_j|) (gamma_4 < 4.01 u, KQ = 5).  The
  distance from the rounded q moves by at most |e_q| (triangle inequality), and its fp32 evaluation (a difference, a
  square and a sum of three non-negative terms, a square root) is within 3.5 u d of it (KD = 4).  So every candidate
  distance is within m(d) = |e_q| + KD u d of float64.  An arg-min is decided when second - best > m(best) + m(second):
  then it must be float64's; an undecided pick must lie within m of the minimum; bitwise-equal targets give bitwise-equal
  distances, so the first index must win (knn_cuda's rule).  The strict keep test d < voxel must equal float64's wherever
  |d - voxel| > m(d); the count lies in [decided kept, decided kept + marginal].  Where every fp32 operation is exact
  (identity pose, an axis offset s: sqrt(fl(s s)) = s) the distance is exactly s, so a source at exactly the voxel is
  dropped and one ulp inside is kept -- a known answer the margin cannot decide.
* SO(2) augmentation.  th = sqrtf(fl(a a)) is within 1.5 u th; sinf / cosf within 2 ulp (KS u of the value) plus
  |cos| dth resp. |sin| dth; the axis a / (th + 1e-6) within 1.5 u th / (th + 1e-6) + 2 u; R_22 = c + wz^2 (1 - c) within
  ec |1 - wz^2| + |1 - c| (2 r_wz + 4 u) + u |R_22| -- a factor 2 on all of it.  The first-order form (1, -a, a) is
  exact.  The branch (theta^2 > fp32(1e-6)) is undecided where |a^2 - fp32(1e-6)| <= 2 u a^2; then either form is
  accepted.  Rotated rows: |err| <= KM u |R| |d| + |dR| |d| (a 3-term dot product with the fp32 R, plus R's own error);
  the rows are also bit for bit the fixed-order product with the returned aug_R, so aug_R is the R that was applied.
  No fp32 angle has fl(a a) equal to fp32(1e-6) (test_taylor_threshold_is_never_hit_exactly), so ">=" for ">" at the
  threshold is an equivalent mutation that no test can catch.
* EquiMatch.  A score is a sum of products; any evaluation order with n rounding steps on the path of a term is within
  gamma_n sum |d1| |d2| (gamma_n = n u / (1 - n u)).  bx_equi_match: n = ceil(C / 32) K L (one lane's sequential sum,
  the product included) + 5 (the xor tree).  The fp32 oracle (an einsum, order unknown): n = C K L.  The arg-max over
  shifts equals float64's where the top gap exceeds twice the row's largest bound; eqv_acc is that arg-max.
* SO(2) label.  Each 3-term product is within KM u sum |a| |b| plus the propagated input error, giving e_u and e_v.  The
  unit projection moves by dp <= |e_vxy| / (|v_xy| - |e_vxy|) + 4 u (the conditioning of the xy projection: singular when
  the target axis nears +-z); the cosine by d_cs <= dp + 2 |e_u| / |u| + 10 u; the angle by d_cs / sin (at the endpoint
  |cs| + d_cs) or, near theta in {0, pi}, (pi / sqrt 2) sqrt(d_cs) (acos is 1/2-Hoelder), plus acosf's 2 ulp and KL u 2 pi
  for fp32(2 pi) and 2 pi - angle.  The label bound is azi_n / 2 pi times that plus KL u azi_n.  Labels are compared
  circularly (0 == azi_n: the sign decision near theta = 0 moves a label across the wrap, not by 2 pi); the sign of
  (u x p)_z is decided where |cz| > |u_xy| dp + |e_u,xy| + 4 u (|u0 p1| + |u1 p0|), and otherwise the mirror label is
  accepted too.  Integer labels equal float64's rounding where the label is more than the bound from a half-integer.
  Where |v_xy| <= 2 |e_vxy| the float64 label is undefined: only a finite label in [0, azi_n), and where the fp32
  projection is exactly 0 the reference's value cos = 0, theta = pi / 2, label azi_n / 4.

Each oracle mutation of MUTATIONS fails its named check (test_mutation_is_caught).  The largest ratios are printed with -s
and recorded in DESIGN.md section 7."""
import numpy as np
import pytest
import torch

from oracle import train_cases as C
from oracle import train_stages as TS
from oracle.train_cases import merge, report

F32 = np.float32


# ------------------------------------------------------------------------------------------------ ground-truth matches
def _gt_group(group):
    cases = C.gt_cases()
    if group == "grid":
        return {k: v for k, v in cases.items() if k.startswith("M")}
    if group == "offsets":
        return {k: v for k, v in cases.items() if k.startswith("offset")}
    return {group: cases[group]}


def check_gt_oracle(group, mutations=()):
    acc = {}
    for name, (src, tgt, T, v) in _gt_group(group).items():
        merge(acc, C.check_gt(src, tgt, T, v, TS.matching_indices(src, tgt, T, v, _mutations=mutations)))
    return acc


@pytest.mark.parametrize("group", ["grid", "dup", "offsets", "voxel_edge"])
def test_gt_oracle_vs_fp64(group):
    """M in {0, 1, 2047, 2048, 2049, 4097} x N in {0, 1, 127, 129, 1023, 1024, 1025, 5000} with a non-identity pose,
    duplicated targets, offsets of 1e2 / 1e3 / 1e4 m and sources at exactly the voxel distance."""
    report(f"gt_matches oracle {group}", check_gt_oracle(group))


def check_voxel_edge(mutations=()):
    src, tgt, T, v, keep = C.gt_voxel_edge_case()
    pairs = TS.matching_indices(src, tgt, T, v, _mutations=mutations)
    C.check_gt(src, tgt, T, v, pairs)
    assert np.array_equal(pairs[:, 0], np.flatnonzero(keep)), "exactly-voxel sources kept or one-ulp-inside sources dropped"
    assert np.array_equal(pairs[:, 1], pairs[:, 0]), "nearest target is the grid point below"


def test_gt_voxel_edge_known_answer():
    check_voxel_edge()


@pytest.mark.parametrize("name", ["C1", "C2"])
def test_gt_oracle_training_clouds(name):
    """The second-level clouds add_training_clouds builds (C2: every 5th source row in float64)."""
    src, tgt, T, v = C.training_pair(name)
    pairs = TS.matching_indices(src, tgt, T, v)
    rows = None if name == "C1" else np.arange(0, len(src), 5)
    out = C.check_gt(src, tgt, T, v, pairs, rows=rows)
    assert len(pairs) > 100
    report(f"gt_matches oracle {name} ({len(src)} x {len(tgt)})", out)


# ------------------------------------------------------------------------------------------------ SO(2) augmentation
def check_aug_oracle(K, P, mutations=()):
    delta, ra, ang = C.aug_case(K, P, seed=K + P)
    d, r, R = TS.so2_augment(delta, ra, ang, _mutations=mutations)
    return C.check_aug(delta, ra, ang, d, r, R)


@pytest.mark.parametrize("K", C.AUG_K)
def test_aug_oracle_vs_fp64(K):
    """P in {1, 255, 256, 257, 1024}; the angles 0, +-1e-4, pi / 2, pi, 3 pi / 2, the largest fp32 below 2 pi and +-6 ulps
    around fp32(1e-3) come first, then the reference's draw."""
    acc = {}
    for P in C.AUG_P:
        merge(acc, check_aug_oracle(K, P))
    report(f"so2_augment oracle K={K}", acc)


def test_taylor_threshold_is_never_hit_exactly():
    """fl(a a) == fp32(1e-6) for no fp32 a (a^2 is monotone, so only the values next to sqrt(1e-6) can come close):
    the kernel's th2 > 1e-6f and kornia's theta^2 > 1e-6 cannot tell ">" from ">="."""
    thr = F32(TS.AUG_THRESHOLD)
    x = F32(np.sqrt(float(thr)))
    for _ in range(64):
        x = np.nextafter(x, F32(0))
    vals = []
    for _ in range(128):
        vals.append(x)
        x = np.nextafter(x, F32(1))
    sq = np.asarray(vals, F32) * np.asarray(vals, F32)
    assert sq.min() < thr < sq.max() and not (sq == thr).any()


# ------------------------------------------------------------------------------------------------ EquiMatch
def _equi_shapes():
    return [(c, k, l) for c in C.EQ_C for k in C.EQ_K for l in C.EQ_L if c * k * l <= C.EQ_LIMIT] + \
        [(32, 6, 32), (6144, 1, 1), (1, 6144, 1)]


def check_equi_oracle(mutations=(), shapes=None, B=8):
    acc = {}
    for C_, K, L in shapes or _equi_shapes():
        for kind in ("unit", "raw", "cancel"):
            d1, d2 = C.equi_case(B, C_, K, L, kind, seed=C_ + K + L)
            got = TS.equi_match(d1, d2, _mutations=mutations).numpy()
            merge(acc, C.check_equi(d1, d2, got, C_ * K * L))
    return acc


def test_equi_oracle_vs_fp64():
    """C in {1, 31, 32, 33, 64}, K in {1, 5, 7}, L in {1, 2, 20, 32} within 48 KB, and C K L exactly at it; unit,
    unnormalised and cancelling maps."""
    report("equi_match oracle", check_equi_oracle())


def test_equi_bound_is_relative_to_the_magnitudes():
    """On cancelling maps the scores are far below sum |d1| |d2|: a bound relative to the row's largest score would be
    meaningless there."""
    d1, d2 = C.equi_case(8, 32, 7, 20, "cancel", seed=3)
    ref = TS.equi_match(d1.double(), d2.double()).abs().max()
    mag = TS.equi_match(d1.double().abs(), d2.double().abs()).max()
    assert ref < 1e-4 * mag


# ------------------------------------------------------------------------------------------------ SO(2) label
def check_label_oracle(kind, azi_n, mutations=(), integer=(True, False), P=4000):
    s, a, b, T, A = C.label_case(kind, P, azi_n, seed=azi_n)
    acc = {}
    for it in integer:
        got = TS.so2_gt(s, a, b, T, azi_n, it, aug_R=A, _mutations=mutations)
        merge(acc, C.check_label(s, a, b, T, azi_n, got, it, aug_R=A))
    return acc


@pytest.mark.parametrize("kind", ["random", "aug", "axis", "align"])
def test_label_oracle_vs_fp64(kind):
    """azi_n in {1, 4, 20, 36}; random frames with and without the augmentation, target axes at and next to +-z, theta = 0
    and pi, labels at k + 1/2 +- a few ulps and angles just below 2 pi."""
    for azi_n in C.GT_AZI:
        out = check_label_oracle(kind, azi_n)
        if kind == "axis":
            assert out["undefined"] > 0
        report(f"so2_gt oracle {kind} azi_n={azi_n}", out)


def test_label_small_counts():
    for P in C.GT_P:
        check_label_oracle("random", 20, P=P)


def test_label_zero_projection_is_a_quarter_turn():
    """Target axis exactly +-z: v_xy = 0 in fp32, F.normalize gives 0, the cosine 0, theta = pi / 2."""
    s, a, b, T, _ = C.label_case("axis", 30, 20, seed=0)
    _, _, _, _, zero = C.label_bound(s, a, b, T, 20)
    assert zero.sum() == 10
    assert (TS.so2_gt(s, a, b, T, 20, True)[zero] == 5).all()
    assert np.abs(TS.so2_gt(s, a, b, T, 20, False)[zero] - 5).max() <= 1e-5


# ------------------------------------------------------------------------------------------------ mutations
MUTATIONS = [
    ("le", lambda m: check_voxel_edge(m)),
    ("last_tie", lambda m: check_gt_oracle("dup", m)),
    ("T_transposed", lambda m: check_gt_oracle("grid", m)),
    ("no_eps", lambda m: check_aug_oracle(700, 1, m)),
    ("transposed", lambda m: check_aug_oracle(700, 1, m)),
    ("shift_plus", lambda m: check_equi_oracle(m, shapes=[(32, 7, 20)])),
    ("sign_inverted", lambda m: check_label_oracle("random", 20, m)),
    ("no_wrap", lambda m: check_label_oracle("random", 20, m)),
    ("aug_untransposed", lambda m: check_label_oracle("aug", 20, m)),
]


@pytest.mark.parametrize("mutation,check", MUTATIONS, ids=[m for m, _ in MUTATIONS])
def test_mutation_is_caught(mutation, check):
    check(())                                            # passes on the oracle as written
    with pytest.raises(AssertionError):
        check((mutation,))


def test_ge_threshold_mutation_is_equivalent():
    """">=" at the Taylor threshold changes no rotation: see test_taylor_threshold_is_never_hit_exactly."""
    a = C.edge_angles()
    assert np.array_equal(TS.aug_rotations(a), TS.aug_rotations(a, ("ge_threshold",)))
