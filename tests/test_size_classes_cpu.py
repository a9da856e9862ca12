"""Size classes of the throughput path: the FPS tier table exported by the library (bx_fps_size_class) and the slot keys of
BufferX under enable_cuda_graphs(..., size_classes=True).  Host-side only: no kernel runs."""
import pytest

# the default launch table of bx_fps_ex (max_cluster 0): the largest point count of every register tier
BOUNDARIES = [4096, 8192, 16384, 24576, 32768, 65536, 131072, 262144, 524288]


@pytest.fixture(scope="module")
def ops():
    from bufferx_b200 import ops
    ops.load_library()
    return ops


def test_size_class_table_boundaries(ops):
    for i, b in enumerate(BOUNDARIES):
        assert ops.fps_size_class(b) == b
        assert ops.fps_size_class(b - 1) == b
        nxt = BOUNDARIES[i + 1] if i + 1 < len(BOUNDARIES) else -1          # beyond 524288 points no launch exists
        assert ops.fps_size_class(b + 1) == nxt
    assert ops.fps_size_class(1) == 4096 and ops.fps_size_class(0) == 0


def test_size_class_is_monotone_and_idempotent(ops):
    prev = 0
    for n in sorted(set(range(1, 140000, 997)) | {9000, 12000, 20000, 30000, 60000, 120000}):
        c = ops.fps_size_class(n)
        assert c >= n and ops.fps_size_class(c) == c and c >= prev
        prev = c


@pytest.mark.parametrize("max_cluster", [2, 4])
def test_size_class_throughput_form(ops, max_cluster):
    """The 2- / 4-CTA form has its own tiers up to 49152 points; a class never crosses a change of launch configuration."""
    per_cta = [4096, 6144, 10240, 12288]
    cl = max_cluster
    expect = [4096, 8192] + [min(p * cl, 49152) for p in per_cta if p * cl > 8192]
    if cl == 2:
        expect += [32768, 65536]          # 24577..49152 points fall back to the latency form's tiers
    for b in expect:
        assert ops.fps_size_class(b, max_cluster) == b
        assert ops.fps_size_class(b - 1, max_cluster) == b
    assert ops.fps_size_class(50000, max_cluster) == 65536


def _model(**kw):
    import bufferx_b200 as bx
    from bufferx_b200.synth import workload_cfg
    cfg = workload_cfg("C2")
    for k, v in kw.items():
        setattr(cfg.match, k, v)
    return bx.BufferX(cfg)


def test_slot_keys():
    m = _model()
    assert m._slot_key(9000, 20000, False) == ((9000, 20000, False, False, None), 9000, 20000, False)     # default: exact shapes
    m.enable_cuda_graphs(True, size_classes=True)
    assert m._slot_key(9000, 20000, False) == ((16384, 24576, False, False, None), 16384, 24576, True)
    assert m._slot_key(16000, 24576, True)[0] == (16384, 24576, True, False, None)
    assert m._slot_key(60000, 30000, True)[0] == (65536, 32768, True, False, None)
    assert m._slot_key(200000, 5000, False)[0] == (262144, 8192, False, False, None)
    # a pair whose larger cloud has more than 200000 points keeps an exact-shape slot
    assert m._slot_key(200001, 5000, False) == ((200001, 5000, False, False, None), 200001, 5000, False)
    assert m._slot_key(5000, 250000, True) == ((5000, 250000, True, False, None), 5000, 250000, False)
    m.enable_cuda_graphs(False)
    assert m._slot_key(9000, 20000, False)[0] == (9000, 20000, False, False, None)


def test_slot_keys_carry_the_early_exit_setting():
    m = _model(enable_early_exit=True, early_exit_min_inliers=7)
    m.enable_cuda_graphs(True, size_classes=True)
    assert m._slot_key(20000, 20000, False)[0] == (24576, 24576, False, True, 7)
