"""CPU-side checks of the tensor-core trainer kind: the 3xTF32 operand split restated in numpy, and the refusal of an unknown kind before
any device is touched."""
import numpy as np
import pytest


def tf32_rna(x):
    """cvt.rna.tf32.f32: round an fp32 value to 10 explicit mantissa bits, ties away from zero (the low 13 bits cleared)"""
    b = np.asarray(x, np.float32).view(np.uint32).astype(np.uint64)
    finite = (b & 0x7F800000) != 0x7F800000
    r = ((b + 0x1000) & 0xFFFFE000).astype(np.uint32)                # add half of the dropped field: ties go away from zero
    return np.where(finite, r, b.astype(np.uint32)).view(np.float32)


def split(x):
    x = np.asarray(x, np.float32)
    big = tf32_rna(x)
    with np.errstate(over="ignore", invalid="ignore"):
        small = tf32_rna((x - big).astype(np.float32))                  # exact in fp32
    return big, small


# the absolute floor: below 2^-126 fp32 (and tf32) values are subnormal, and a tf32 subnormal keeps 10 bits, spacing 2^-136, so the
# small term rounds to within 2^-137
FLOOR = 2.0 ** -137
# the largest value the split holds: above (2 - 2^-11) 2^127 (0.02 % below fp32's largest) the big term rounds to infinity
SPLIT_MAX = (2.0 - 2.0 ** -11) * 2.0 ** 127


def edge_values():
    p2 = np.float32(2.0) ** np.arange(-149, 128, dtype=np.float32)
    halfway = (p2[:-1] * np.float32(1 + 2.0 ** -11)).astype(np.float32)        # exactly halfway between two tf32 values
    halfway2 = (p2[:-1] * np.float32(1 + 3 * 2.0 ** -11)).astype(np.float32)
    near = (p2[:-1] * np.float32(1 + 2.0 ** -11 + 2.0 ** -23)).astype(np.float32)
    special = np.array([0.0, -0.0, 1e-38, -1e-38, 3e38, -3e38, 1e-30, 1e-45, 2.0 ** -140, 1.0 - 2.0 ** -24, 3.4e38], np.float32)
    v = np.concatenate([p2, halfway, halfway2, near, special])
    return np.concatenate([v, -v]).astype(np.float32)


@pytest.mark.parametrize("which", ["random", "edges"])
def test_split_error_bound(which):
    """|x - big - small| <= 2^-22 |x| + the subnormal floor, and big, small are tf32 values (low 13 bits zero); |x| < SPLIT_MAX"""
    if which == "random":
        rng = np.random.default_rng(0)
        x = (rng.standard_normal(200000) * np.exp(rng.uniform(-80, 80, 200000))).astype(np.float32)
    else:
        x = edge_values()
    big, small = split(x)
    assert ((big.view(np.uint32) & 0x1FFF) == 0).all() and ((small.view(np.uint32) & 0x1FFF) == 0).all()
    err = np.abs(x.astype(np.float64) - big.astype(np.float64) - small.astype(np.float64))
    bound = 2.0 ** -22 * np.abs(x.astype(np.float64)) + FLOOR
    assert (err <= bound).all(), x[np.argmax(err / bound)]
    # the bound is tight within a factor of two: a single tf32 term would miss it by ~2^10
    one = np.abs(x.astype(np.float64) - big.astype(np.float64))
    assert (one > bound).any()


def test_split_overflows_only_next_to_the_fp32_maximum():
    big, _ = split(np.array([np.nextafter(np.float32(SPLIT_MAX), np.float32(0)), 3.4028235e38], np.float32))
    assert np.isfinite(big[0]) and np.isinf(big[1])


def test_round_to_nearest_ties_away():
    one = np.float32(1.0)
    ulp = np.float32(2.0 ** -10)
    assert tf32_rna(one + ulp / 2) == one + ulp                         # halfway rounds away from zero
    assert tf32_rna(-(one + ulp / 2)) == -(one + ulp)
    assert tf32_rna(np.float32(one + ulp / 2 - 2.0 ** -23)) == one
    assert tf32_rna(np.float32(0.0)) == 0 and np.signbit(tf32_rna(np.float32(-0.0)))


def test_unknown_trainer_kind_refused_before_the_device():
    from tetris_mcts_b200.model import trainer as T
    called = []
    orig = T._lib
    T._lib = lambda: called.append(1) or orig()
    try:
        with pytest.raises(ValueError):
            T.Trainer(np.zeros(478342, np.float32), kind="bogus")
    finally:
        T._lib = orig
    assert not called


def test_train_kind_flag():
    from tetris_mcts_b200 import play_batched as PB
    assert PB.parse_args([]).train_kind == "fp64"
    assert PB.parse_args(["--train_kind", "tc"]).train_kind == "tc"
    with pytest.raises(SystemExit):
        PB.parse_args(["--train_kind", "bf16"])
