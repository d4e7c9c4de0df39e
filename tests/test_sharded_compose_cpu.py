"""CPU: the composer's entries for Gaussian sharding (include/sgr.h sgr_compose_pose_rows, sgr_compose_backward_rows,
sgr_compose_pose_finalize, sgr_compose_pose_reduce_peers) validate their arguments before anything is enqueued, and a numpy restatement of
compose.cu's finalize shows why "sum the ranks' accumulator rows, then finalize" is the frame's gradient: the finalize is one fixed linear
map of a row (coefficients from the pose and the correction only), so finalizing the sum of rank shares equals finalizing the whole
frame's rows, up to the order of the additions."""
import ctypes as C

import numpy as np
import torch

import street_gaussians_b200 as sgb
from street_gaussians_b200 import _capi
from street_gaussians_b200 import sharded as SH

OK = C.c_void_p(1 << 20)  # a 16-byte aligned address: validation fails before anything dereferences it


def _err():
    return _capi.lib().sgr_last_error().decode()


def _segs(counts):
    segs = (_capi.SgrSegment * len(counts))()
    start = 0
    for k, n in enumerate(counts):
        s = segs[k]
        s.start, s.count, s.fourier_dim, s.posed = start, n, 1 if k == 0 else 5, int(k > 0)
        s.xyz = s.rotation = s.scaling = s.opacity = s.features_dc = s.features_rest = OK.value if n else None
        start += n
    return segs


def test_pose_rows():
    L = _capi.lib()
    assert L.sgr_compose_pose_rows(9, 0) == 9 and L.sgr_compose_pose_rows(9, 1) == 10 and L.sgr_compose_pose_rows(0, 1) == 0


def test_backward_rows_validates_before_launch():
    L = _capi.lib()
    segs = _segs([10, 0, 4])
    grads = (_capi.SgrSegmentGrads * 3)()
    for k in (0, 2):
        g = grads[k]
        g.xyz = g.rotation = g.scaling = g.opacity = g.features_dc = g.features_rest = OK.value
    up = [OK] * 5

    def call(segs=segs, grads=grads, n=3, M=16, poses=OK, corr=OK, acc=OK, nbytes=4 * 64, flip=None, fq=None, up=up):
        return L.sgr_compose_backward_rows(segs, grads, n, M, poses, OK, flip, fq, corr, *up, acc, nbytes, None)

    assert call(n=0) == -1 and "empty" in _err()
    assert call(M=0) == -1 and "SH coefficients" in _err()
    assert call(acc=None) == -1 and "NULL pointer" in _err()
    assert call(poses=None) == -1 and "NULL pointer" in _err()
    assert call(up=[OK, None, OK, OK, OK]) == -1 and "upstream" in _err()
    assert call(flip=OK) == -1 and "flip_quat" in _err()
    g1 = (_capi.SgrSegmentGrads * 3)()
    assert call(grads=g1) == -1 and "segment 0 has a NULL gradient" in _err()
    # 3 segments + the correction's row = 4 rows of 64 bytes; 3 rows without a correction
    assert call(nbytes=4 * 64 - 1) == -3 and "256 needed" in _err()
    assert call(corr=None, nbytes=3 * 64 - 4) == -3 and "192 needed" in _err()


def test_finalize_and_peer_reduce_validate_before_launch():
    L = _capi.lib()
    segs = _segs([10, 0, 4])

    def fin(segs=segs, n=3, poses=OK, corr=OK, acc=OK, nbytes=4 * 64, dposes=OK, dcorr=OK):
        return L.sgr_compose_pose_finalize(segs, n, poses, corr, acc, nbytes, dposes, dcorr, None)

    assert fin(segs=None) == -1 and "empty" in _err()
    assert fin(n=0) == -1 and "empty" in _err()
    assert fin(acc=None) == -1 and "NULL pointer" in _err()
    assert fin(dposes=None) == -1 and "NULL pointer" in _err()
    assert fin(dcorr=None) == -1 and "without dcorrection" in _err()
    assert fin(corr=None) == -1 and "without bkgd_correction" in _err()
    assert fin(nbytes=64) == -3 and "needed" in _err()

    pe = _capi.SgrPeers()

    def red(peers=pe, nbytes=4 * 64):
        return L.sgr_compose_pose_reduce_peers(C.byref(peers) if peers is not None else None, segs, 3, OK, OK, OK, nbytes, OK, OK, None)

    assert red(peers=None) == -1 and "peers is NULL" in _err()
    assert red(nbytes=3 * 64) == -3 and "needed" in _err()
    pe.world, pe.rank, pe.chunk = 0, 0, 8
    assert red() == -1 and "bad peer table" in _err()
    pe.world, pe.rank = 2, 1
    assert red() == -1 and "entry 0 is NULL" in _err()
    for p in range(2):
        pe.records[p], pe.radii[p], pe.grad2d[p] = OK.value, OK.value, OK.value
    assert red() == -1 and "entry 0 has no composer accumulator section" in _err()
    pe.pose_acc[0] = pe.pose_acc[1] = OK.value
    assert red() == -1 and "entry 0 has no barrier pad" in _err()


def test_peer_workspace_wires_the_accumulator_section():
    """PeerWorkspace.emulate on CPU buffers: every rank's pose_acc entry points at the section of every rank, which sits after the feature
    sections, 256-byte aligned, and holds POSE_ACC_ROWS rows of 16 floats before the barrier pad."""
    st = sgb.GaussianRasterizationSettings(96, 128, 0.5, 0.4, torch.zeros(3), 1.0, torch.eye(4), torch.eye(4), 0, torch.zeros(3), False, False)
    for S in (0, 5):
        wss = SH.PeerWorkspace.emulate(st, 11, 3, torch.device("cpu"), S)
        bases = [ws.buf.data_ptr() for ws in wss]
        for ws in wss:
            assert ws.off_pose % 256 == 0 and ws.off_pose >= ws.off_gsem + 4 * ws.P_total * S
            assert ws.off_flags >= ws.off_pose + 64 * _capi.POSE_ACC_ROWS and ws.total == ws.off_flags + 256
            assert [ws.peers.pose_acc[p] for p in range(3)] == [b + ws.off_pose for b in bases]


# ---- numpy restatement of compose_pose_finalize_kernel (compose.cu) ---------------------------------------------------------------
def _matrix_path(a, q):
    n = np.sqrt((q * q).sum())
    w, x, y, z = q / n
    G = a[:9].reshape(3, 3)
    dw = 2 * (-z * G[0, 1] + y * G[0, 2] + z * G[1, 0] - x * G[1, 2] - y * G[2, 0] + x * G[2, 1])
    dx = 2 * (y * G[0, 1] + z * G[0, 2] + y * G[1, 0] - 2 * x * G[1, 1] - w * G[1, 2] + z * G[2, 0] + w * G[2, 1] - 2 * x * G[2, 2])
    dy = 2 * (-2 * y * G[0, 0] + x * G[0, 1] + w * G[0, 2] + x * G[1, 0] + z * G[1, 2] - w * G[2, 0] + z * G[2, 1] - 2 * y * G[2, 2])
    dz = 2 * (-2 * z * G[0, 0] - w * G[0, 1] + x * G[0, 2] + w * G[1, 0] - 2 * z * G[1, 1] + y * G[1, 2] + x * G[2, 0] + y * G[2, 1])
    d = np.array([dw, dx, dy, dz])
    u = np.array([w, x, y, z])
    return (d - u * (u * d).sum()) / n


def _finalize(acc, poses, posed, corr):
    """dposes [nseg, 7] and dcorrection [7] from accumulator rows acc [nseg + 1, 16] (the last row: the correction's)."""
    dposes = np.zeros((len(posed), 7))
    for s, p in enumerate(posed):
        if p:
            dposes[s, :4] = acc[s, 9:13] + _matrix_path(acc[s], poses[s, :4])
            dposes[s, 4:] = acc[s, 13:16]
    a = acc[-1]
    c = corr[:4]
    cn = np.sqrt((c * c).sum())
    qc = c / max(cn, 1e-12)
    gq = a[9:13] + _matrix_path(a, qc)
    dq = (gq - qc * (qc * gq).sum()) / cn if cn >= 1e-12 else gq / 1e-12
    return dposes, np.concatenate([dq, a[13:16]])


def test_sum_then_finalize_equals_finalize_of_the_whole():
    """Rank shares of every accumulator row (some ranks holding nothing of a segment, as rebalance can leave them) summed in rank order and
    finalized give the finalize of the whole frame's rows, to float64 rounding; the finalize of each share alone, summed, too (linearity).
    Dropping a share or skipping the finalize does not."""
    rng = np.random.default_rng(3)
    for world in (1, 2, 3, 5, 8):
        nseg = 9
        posed = [0] + [1] * 8
        poses = rng.standard_normal((nseg, 7))
        corr = np.concatenate([[1.0, 0, 0, 0] + 0.1 * rng.standard_normal(4), rng.standard_normal(3)])
        shares = rng.standard_normal((world, nseg + 1, 16))
        shares[rng.random((world, nseg + 1)) < 0.3] = 0.0  # segments with no rows on a rank
        whole = shares.sum(0)
        summed = np.zeros_like(whole)
        for r in range(world):
            summed = summed + shares[r]
        dp_whole, dc_whole = _finalize(whole, poses, posed, corr)
        dp_sum, dc_sum = _finalize(summed, poses, posed, corr)
        assert np.allclose(dp_sum, dp_whole, rtol=0, atol=1e-12) and np.allclose(dc_sum, dc_whole, rtol=0, atol=1e-12)
        parts = [_finalize(shares[r], poses, posed, corr) for r in range(world)]
        assert np.allclose(sum(p[0] for p in parts), dp_whole, atol=1e-12) and np.allclose(sum(p[1] for p in parts), dc_whole, atol=1e-12)
        if world > 1:
            big = int(np.abs(shares).sum((1, 2)).argmax())
            dp_drop, dc_drop = _finalize(summed - shares[big], poses, posed, corr)
            assert not (np.allclose(dp_drop, dp_whole, atol=1e-6) and np.allclose(dc_drop, dc_whole, atol=1e-6))
        raw = np.concatenate([whole[1:nseg, 9:13], whole[1:nseg, 13:16]], 1)
        assert not np.allclose(raw, dp_whole[1:], atol=1e-6)
