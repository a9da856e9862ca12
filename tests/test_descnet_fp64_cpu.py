"""The descriptor network (a6-a9) against float64 without a GPU: the float64 oracle functions (oracle.desc_fp64,
oracle.pnt_fp64) against the fp32 oracle, the presplit image helpers (ops.sd_pack / ops.sd_unpack), and oracle.spt on the
hand-built edge patches (oracle/spt_cases.py) against a plain NumPy voxel-major ball query, which pins the oracle before the
kernel is held to it bit for bit (tests/test_descnet_fp64_gpu.py)."""
import numpy as np
import pytest
import torch

from oracle import spt_cases


@pytest.fixture(scope="module")
def sd():
    import bufferx_b200 as bx
    from bufferx_b200.synth import init_synthetic_weights, workload_cfg
    model = init_synthetic_weights(bx.BufferX(workload_cfg("C2")))
    return {k: v.detach().clone() for k, v in model.state_dict().items()}


def ball_query_np(delta, rad_n, azi_n, ele_n, rho, nv):
    """Voxel-major restatement of the reference's sphere query + var_to_invar: for every voxel, the first nv points (index
    order) with ((dx^2 + dy^2) + dz^2) < rho^2 in fp32, padding slots repeat the first, slot 0 holding index 0 and the
    padding slots are zero, the others de-rotated by (cos, sin) of -a 2 pi / azi_n in fp32."""
    from oracle import oracle as O
    vox, rot = O.voxel_table(rad_n, azi_n, ele_n), O.derot_table(azi_n)
    K, P, _ = delta.shape
    V = len(vox)
    r2 = np.float32(rho) * np.float32(rho)
    vidx = np.zeros((K, V, nv), np.int32)
    inv = np.zeros((K, V, nv, 3), np.float32)
    for k in range(K):
        p = delta[k]
        dx, dy, dz = vox[:, None, 0] - p[None, :, 0], vox[:, None, 1] - p[None, :, 1], vox[:, None, 2] - p[None, :, 2]
        hit = ((dx * dx + dy * dy) + dz * dz) < r2
        for v in range(V):
            idx = np.flatnonzero(hit[v])[:nv]
            if len(idx) == 0:
                continue
            row = np.full(nv, idx[0], np.int32)
            row[:len(idx)] = idx
            vidx[k, v] = row
            cs, sn = rot[v % azi_n]
            live = row != row[0]
            live[0] = row[0] != 0
            x, y, z = p[row, 0], p[row, 1], p[row, 2]
            q = np.stack([x * cs + y * (-sn), x * sn + y * cs, z], axis=1)
            inv[k, v] = np.where(live[:, None], q, np.float32(0))
    return vidx, inv


@pytest.mark.parametrize("P,nv,rho,table", [(1, 10, 0.8 / 3, (3, 7, 20)), (33, 10, 0.8 / 3, (3, 7, 20)),
                                            (100, 16, 0.5, (3, 7, 20)), (31, 1, 0.1, (2, 5, 12)),
                                            (512, 10, 0.8 / 3, (4, 9, 24))])
def test_oracle_spt_equals_voxel_major_ball_query(oracle, P, nv, rho, table):
    rad_n, ele_n, azi_n = table
    delta = spt_cases.spt_patches(P, rad_n, azi_n, ele_n, rho, seed=P)
    inv, vidx = oracle.spt(delta, rad_n, azi_n, ele_n, rho, nv)
    evidx, einv = ball_query_np(delta, rad_n, azi_n, ele_n, rho, nv)
    assert (vidx == evidx).all()
    assert (inv.view(np.int32) == einv.view(np.int32)).all()             # bit for bit, signed zeros included
    # the cases are there: balls with more than 16 hits, exact r^2 boundaries, empty and full voxels
    hits = np.zeros(vidx.shape[:2], np.int64)
    vox = oracle.voxel_table(rad_n, azi_n, ele_n)
    r2 = np.float32(rho) * np.float32(rho)
    on = 0
    for k in range(delta.shape[0]):
        d2 = np.stack([spt_cases.d2_f32(c, delta[k]) for c in vox])
        hits[k] = (d2 < r2).sum(axis=1)
        on += int((d2 == r2).sum())
    assert on > 0 and (hits == 0).any()
    if P >= 100:
        assert hits.max() > 16
    assert (delta[0] == 0).all() and (delta[2, 0] == 0).all() and (delta[1, 0] != 0).any()


def test_pnt_fp64_against_the_fp32_oracle(oracle, sd):
    delta = spt_cases.spt_patches(100, seed=3)
    inv, vidx = oracle.spt(delta)
    with torch.no_grad():
        f32 = oracle.pnt_max(torch.from_numpy(inv), sd).double()
    f64, absref = oracle.pnt_fp64(delta, vidx, sd, absref=True)
    assert f64.dtype == torch.float64 and f64.shape == (delta.shape[0], 16, 420)
    assert ((f32 - f64).abs() <= 2e-6 * absref).all()
    assert (absref >= f64).all()
    # the all-zero patch: every sample is a zeroed slot -> relu(b) everywhere
    assert torch.equal(f64[0], f64[0, :, :1].expand(16, 420))


def test_desc_fp64_against_the_fp32_oracle(oracle, sd):
    delta = spt_cases.spt_patches(100, seed=4)
    inv, vidx = oracle.spt(delta)
    feat = oracle.pnt_fp64(delta, vidx, sd).float()
    K = feat.shape[0]
    d64, aux = oracle.desc_fp64(feat, sd, keep=True)
    assert torch.equal(oracle.desc_fp64(feat, sd), d64)
    acts = aux["acts"]
    assert [tuple(a.shape[1:]) for a in acts] == [(64, 7, 20), (64, 7, 20), (128, 7, 20), (128, 7, 20), (64, 7, 20),
                                                  (64, 7, 20), (32, 7, 20), (32, 7, 20)]
    assert all(a.dtype == torch.float64 for a in acts) and all((a >= 0).all() for a in acts[:7])
    with torch.no_grad():
        x32 = oracle.cyl_net(feat.view(K, 16, 3, 7, 20), sd)
        d32, e32 = oracle.pool_desc(x32, sd)
    x = acts[7]
    scale = x.abs().amax(dim=(1, 2, 3)).view(K, 1, 1, 1)
    assert ((x32.double() - x).abs() <= 1e-5 * scale).all()
    assert ((e32.double() - aux["equi"]).abs() <= 1e-5).all()
    pooled = aux["pooled"]
    assert torch.allclose(pooled, (x * aux["att"]).mean(dim=(2, 3)), rtol=1e-12, atol=0)
    nrm = pooled.norm(dim=1)
    assert torch.allclose(d64, pooled / nrm.clamp(min=1e-12)[:, None], rtol=1e-12, atol=0)
    ok = nrm > 1e-3 * nrm.max()                   # well-conditioned rows: the fp32 oracle to fp32 grade
    assert ((d32.double() - d64).abs().max(dim=1).values[ok] <= 1e-5).all()


@pytest.mark.parametrize("C", [16, 48, 64])
@pytest.mark.parametrize("n", [1, 3])
def test_sd_pack_unpack_round_trip(C, n):
    from bufferx_b200 import ops
    g = torch.Generator().manual_seed(C + n)
    x = torch.randn(n, C, 7, 20, generator=g) * torch.logspace(-6, 4, C).view(1, C, 1, 1)
    img = ops.sd_pack(x)
    rows = ops.conv_sd_rows(n)
    assert img.shape == (C // 16, 4, rows, 8) and img.dtype == torch.float16
    val, xp = ops.sd_unpack(img, n)
    # hi + lo * 2^-11 keeps 22 bits; below fp16's normal range the lo part keeps 2^-35 absolute
    assert ((val.double() - x.double()).abs() <= 2.0 ** -22 * x.double().abs() + 2.0 ** -35).all()
    assert (xp[:, :, 0] == 0).all()                                         # the zero row above the first elevation
    assert torch.equal(xp[:, :, 1:, 0], xp[:, :, 1:, 20]) and torch.equal(xp[:, :, 1:, 21], xp[:, :, 1:, 1])   # wrap columns
    assert (img[:, :, n * 176:].float() == 0).all()                         # the row after the last sample, and the tail
    # chunk c holds channels 16c..16c+15: for the 48-channel CYL3D input, chunk r = radial slice r of [n,16,3,7,20]
    for c in range(C // 16):
        assert torch.equal(ops.sd_pack(x[:, 16 * c:16 * c + 16].contiguous()).view(torch.int16), img[c:c + 1].view(torch.int16))
