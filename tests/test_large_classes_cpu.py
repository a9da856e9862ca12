"""Size classes for clouds above 200000 points (enable_cuda_graphs(..., size_classes=True, large_classes=True)): the capacity
ladder exported by the library (bx_fps_large_size_class) and the slot keys it gives.  Host-side only: no kernel runs."""
import pytest

LIMIT = 1638400
PER_CTA = 18432          # bx_fps_large: points per CTA of the grid-wide FPS kernel


@pytest.fixture(scope="module")
def ops():
    from bufferx_b200 import ops
    ops.load_library()
    return ops


def _boundaries(ops):
    """The class capacities above 200000 points, in order."""
    caps, n = [], 200001
    while n <= LIMIT:
        c = ops.fps_large_size_class(n)
        caps.append(c)
        n = c + 1
    return caps


def test_ladder_covers_every_large_count(ops):
    caps = _boundaries(ops)
    assert caps[-1] == LIMIT
    assert caps == sorted(set(caps))
    lo = 200000
    for c in caps:
        # every count of the class maps to the class, the class is a fixed point, and the next count starts a new class
        for n in (lo + 1, (lo + 1 + c) // 2, c):
            assert ops.fps_large_size_class(n) == c
        assert ops.fps_large_size_class(c + 1) != c
        lo = c
    assert ops.fps_large_size_class(LIMIT + 1) == -1


def test_ladder_above_the_cluster_limit(ops):
    """Above 524288 points: multiples of the grid kernel's 18432 points per CTA (the top class is the 1638400-point limit)
    with at most 25 % padding over the smallest cloud of the class."""
    caps = [c for c in _boundaries(ops) if c > ops.FPS_MAX_POINTS]
    assert len(caps) <= 8
    lo = ops.FPS_MAX_POINTS
    for c in caps:
        assert c % PER_CTA == 0 or c == LIMIT
        assert c <= 1.25 * (lo + 1), (lo, c)
        lo = c
    assert -(-LIMIT // PER_CTA) <= 96          # the grid kernel's candidate reduction


def test_ladder_is_monotone_and_idempotent(ops):
    prev = 0
    for n in sorted(set(range(1, LIMIT + 1, 4999)) | {200000, 200001, 524288, 524289, LIMIT}):
        c = ops.fps_large_size_class(n)
        assert c >= n and ops.fps_large_size_class(c) == c and c >= prev
        prev = c


def test_ladder_equals_fps_size_class_up_to_the_cluster_limit(ops):
    for n in [0, 1, 4096, 4097, 9000, 30000, 49152, 60000, 131073, 200000, 200001, 262145, 524288]:
        assert ops.fps_large_size_class(n) == ops.fps_size_class(n)


def _model(**kw):
    import bufferx_b200 as bx
    from bufferx_b200.synth import workload_cfg
    cfg = workload_cfg("C2")
    for k, v in kw.items():
        setattr(cfg.match, k, v)
    return bx.BufferX(cfg)


def test_slot_keys_with_large_classes(ops):
    m = _model()
    m.enable_cuda_graphs(True, size_classes=True, large_classes=True)
    c = ops.fps_large_size_class
    # both clouds large
    assert m._slot_key(700000, 600000, False) == ((c(700000), c(600000), False, False, None), c(700000), c(600000), True)
    assert m._slot_key(700000, 600000, False)[0] == (792576, 645120, False, False, None)
    assert m._slot_key(1638400, 1000000, True)[0] == (LIMIT, 1216512, True, False, None)
    # mixed large and small
    assert m._slot_key(900000, 20000, True)[0] == (976896, 24576, True, False, None)
    assert m._slot_key(5000, 250000, True) == ((8192, 262144, True, False, None), 8192, 262144, True)
    assert m._slot_key(5000, 300000, True)[0] == (8192, 524288, True, False, None)
    # at the sub-sample boundary and at the cluster limit
    assert m._slot_key(200000, 5000, False)[0] == (262144, 8192, False, False, None)
    assert m._slot_key(200001, 5000, False) == ((262144, 8192, False, False, None), 262144, 8192, True)
    assert m._slot_key(524288, 524289, False)[0] == (524288, 645120, False, False, None)
    assert m._slot_key(524289, 524288, False)[0] == (645120, 524288, False, False, None)
    # pairs of different sizes share a class
    assert m._slot_key(600000, 300000, False)[0] == m._slot_key(640000, 500000, False)[0]
    # small pairs keep today's classes
    assert m._slot_key(9000, 20000, False) == ((16384, 24576, False, False, None), 16384, 24576, True)


def test_slot_keys_without_large_classes_are_unchanged():
    """The keys of test_size_classes_cpu.py::test_slot_keys, also after the flag has been on and off again."""
    m = _model()
    m.enable_cuda_graphs(True, size_classes=True, large_classes=True)
    m.enable_cuda_graphs(True, size_classes=True)
    assert m._slot_key(9000, 20000, False) == ((16384, 24576, False, False, None), 16384, 24576, True)
    assert m._slot_key(200000, 5000, False)[0] == (262144, 8192, False, False, None)
    assert m._slot_key(200001, 5000, False) == ((200001, 5000, False, False, None), 200001, 5000, False)
    assert m._slot_key(5000, 250000, True) == ((5000, 250000, True, False, None), 5000, 250000, False)
    assert m._slot_key(700000, 600000, True) == ((700000, 600000, True, False, None), 700000, 600000, False)
    m.enable_cuda_graphs(True)
    assert m._slot_key(700000, 600000, True) == ((700000, 600000, True, False, None), 700000, 600000, False)


def test_large_classes_need_size_classes():
    m = _model()
    with pytest.raises(ValueError, match="size_classes"):
        m.enable_cuda_graphs(True, large_classes=True)


def test_large_class_keys_carry_the_early_exit_setting():
    m = _model(enable_early_exit=True, early_exit_min_inliers=7)
    m.enable_cuda_graphs(True, size_classes=True, large_classes=True)
    assert m._slot_key(700000, 20000, False)[0] == (792576, 24576, False, True, 7)
