"""CPU-side checks of the drop-in boundary: the C-ABI library loads and exports every symbol include/sgr.h declares,
the size queries work without a GPU, and the Python surface mirrors the reference API."""
import ctypes as C
import inspect
import os
import re

import pytest
import torch

import street_gaussians_b200 as sgb
from street_gaussians_b200 import _capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    src = open(os.path.join(ROOT, "include", "sgr.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(sgr_[a-z0-9_]+)\s*\(", src)) - {"sgr_alloc_fn"})


def test_library_exports_every_declared_symbol():
    lib = C.CDLL(_capi.LIB_PATH)
    syms = declared_symbols()
    assert len(syms) >= 12
    for s in syms:
        assert hasattr(lib, s), f"libsgr.so does not export {s}"
    assert sorted(_capi.SYMBOLS) == syms


def test_abi_version_and_sizes_no_gpu():
    L = _capi.lib()
    assert L.sgr_abi_version() == _capi.ABI_VERSION
    fr = _capi.SgrFrame()
    fr.P, fr.width, fr.height, fr.D, fr.M = 1000, 640, 480, 3, 16
    fr.tan_fovx, fr.tan_fovy, fr.scale_modifier = 0.5, 0.4, 1.0
    g, i = C.c_size_t(), C.c_size_t()
    assert L.sgr_state_sizes(C.byref(fr), C.byref(g), C.byref(i)) == 0
    assert g.value >= 1000 * 48 and g.value % 256 == 0
    assert i.value >= 640 * 480 * 4
    assert L.sgr_binning_bytes(0) > 0
    assert L.sgr_binning_bytes(1000) >= 1000 * 16
    # invalid frame -> error code + message, no crash
    fr.width = 0
    assert L.sgr_state_sizes(C.byref(fr), C.byref(g), C.byref(i)) == -1
    assert b"bad sizes" in L.sgr_last_error()
    fr.width = 640
    fr.row_begin, fr.row_end, fr.row_step = 5, 2, 1
    assert L.sgr_state_sizes(C.byref(fr), C.byref(g), C.byref(i)) == -1
    assert b"band" in L.sgr_last_error()
    assert L.sgr_knn_scratch_bytes(1000) > 1000 * 16


def test_settings_fields_match_reference_order():
    assert sgb.GaussianRasterizationSettings._fields == (
        "image_height", "image_width", "tanfovx", "tanfovy", "bg", "scale_modifier", "viewmatrix", "projmatrix", "sh_degree",
        "campos", "prefiltered", "debug")


def test_rasterizer_signature_matches_reference():
    sig = inspect.signature(sgb.GaussianRasterizer.forward)
    assert list(sig.parameters)[1:] == ["means3D", "means2D", "opacities", "shs", "colors_precomp", "scales", "rotations",
                                        "cov3D_precomp", "semantics"]
    assert all(sig.parameters[k].default is None for k in ("shs", "colors_precomp", "scales", "rotations", "cov3D_precomp", "semantics"))
    sig = inspect.signature(sgb.rasterize_gaussians)
    assert list(sig.parameters) == ["means3D", "means2D", "sh", "colors_precomp", "semantics", "opacities", "scales", "rotations",
                                    "cov3Ds_precomp", "raster_settings"]
    sig = inspect.signature(sgb.GaussianRasterizer.visible_filter)
    assert list(sig.parameters)[1:] == ["means3D", "scales", "rotations", "cov3D_precomp"]
    assert hasattr(sgb.GaussianRasterizer, "markVisible")


def _settings():
    return sgb.GaussianRasterizationSettings(16, 16, 0.5, 0.5, torch.zeros(3), 1.0, torch.eye(4), torch.eye(4), 0, torch.zeros(3), False, False)


def test_argument_validation_matches_reference_messages():
    r = sgb.GaussianRasterizer(_settings())
    m = torch.zeros(4, 3)
    with pytest.raises(Exception, match="excatly one of either SHs or precomputed colors"):
        r(m, None, torch.zeros(4, 1), scales=torch.ones(4, 3), rotations=torch.ones(4, 4))
    with pytest.raises(Exception, match="excatly one of either SHs or precomputed colors"):
        r(m, None, torch.zeros(4, 1), shs=torch.zeros(4, 1, 3), colors_precomp=torch.zeros(4, 3), scales=torch.ones(4, 3), rotations=torch.ones(4, 4))
    with pytest.raises(Exception, match="exactly one of either scale/rotation pair or precomputed 3D covariance"):
        r(m, None, torch.zeros(4, 1), shs=torch.zeros(4, 1, 3))
    with pytest.raises(Exception, match="exactly one of either scale/rotation pair or precomputed 3D covariance"):
        r(m, None, torch.zeros(4, 1), shs=torch.zeros(4, 1, 3), scales=torch.ones(4, 3), rotations=torch.ones(4, 4), cov3D_precomp=torch.zeros(4, 6))


def test_cpu_tensors_fail_loudly_no_fallback():
    """The product path must not silently compute on the CPU."""
    r = sgb.GaussianRasterizer(_settings())
    with pytest.raises(_capi.SgrError, match="no CPU fallback"):
        r(torch.zeros(4, 3), None, torch.zeros(4, 1), shs=torch.zeros(4, 1, 3), scales=torch.ones(4, 3), rotations=torch.ones(4, 4))
    with pytest.raises(_capi.SgrError):
        sgb.distCUDA2(torch.zeros(4, 3))
    with pytest.raises(RuntimeError, match=r"\(num_points, 3\)"):
        r(torch.zeros(4, 2), None, torch.zeros(4, 1), shs=torch.zeros(4, 1, 3), scales=torch.ones(4, 3), rotations=torch.ones(4, 4))


def test_product_never_imports_oracle():
    """oracle/ is test infrastructure: no module of the product package may reference it."""
    pkg = os.path.join(ROOT, "street_gaussians_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                txt = open(os.path.join(dirpath, f)).read()
                assert "import oracle" not in txt and "from oracle" not in txt and "sgr_oracle" not in txt, f


def test_shims_resolve_to_this_package():
    import importlib
    import sys
    sgb.install_shims()
    dgr = importlib.import_module("diff_gaussian_rasterization")
    assert dgr.GaussianRasterizer is sgb.GaussianRasterizer
    assert dgr.GaussianRasterizationSettings is sgb.GaussianRasterizationSettings
    knn = importlib.import_module("simple_knn._C")
    assert knn.distCUDA2 is sgb.distCUDA2
    for n in ("diff_gaussian_rasterization", "simple_knn", "simple_knn._C"):
        sys.modules.pop(n, None)


def test_band_helpers():
    from street_gaussians_b200.sharded import band_of_rows, contiguous_band, cyclic_band
    H = 1280  # 80 tile rows
    for world in (1, 2, 4, 8, 3):
        for layout, mk in (("cyclic", cyclic_band), ("contiguous", contiguous_band)):
            cover = torch.zeros(H, dtype=torch.int32)
            for r in range(world):
                cover += band_of_rows(H, r, world, layout).int()
            assert (cover == 1).all(), (world, layout)
    b = cyclic_band(100, 3, 8)  # 7 tile rows, rank 3 owns row 3 only
    assert (b.begin, b.end, b.step) == (3, 7, 8)
    assert cyclic_band(16, 5, 8).end == 0  # more ranks than rows -> empty band


def test_debug_mode_dumps_inputs_like_the_reference(tmp_path, monkeypatch):
    """debug=True: a failing forward leaves snapshot_fw.dump with the 20 arguments of the reference's
    _C.rasterize_gaussians call (DGR/diff_gaussian_rasterization/__init__.py:87-94)."""
    monkeypatch.chdir(tmp_path)
    st = _settings()._replace(debug=True)
    r = sgb.GaussianRasterizer(st)
    with pytest.raises(_capi.SgrError):
        r(torch.zeros(4, 3), None, torch.zeros(4, 1), shs=torch.zeros(4, 1, 3), scales=torch.ones(4, 3), rotations=torch.ones(4, 4))
    dump = torch.load(tmp_path / "snapshot_fw.dump")
    assert len(dump) == 20 and dump[1].shape == (4, 3) and dump[-1] is True


def test_instance_capacity_bookkeeping():
    cap = sgb.InstanceCapacity(headroom=1.5)
    assert cap.capacity is None
    cap.observe(1000)
    assert cap.capacity == 1500 + 4096
    cap.observe(10)          # never shrinks
    assert cap.capacity == 1500 + 4096
    cap.check()              # nothing pending: no-op


class _FakeEvent:
    def __init__(self, done=True):
        self.done, self.waited = done, False

    def query(self):
        return self.done

    def synchronize(self):
        self.waited, self.done = True, True


def _status(R, overflow=0, emitted=0, n_sel=0, timed_out=0):
    return torch.tensor([R, overflow, emitted, n_sel, timed_out, 0, 0, 0], dtype=torch.int32)


def test_instance_capacity_async_status_protocol():
    """InstanceCapacity.check(): frames are examined in submission order once their status has arrived; an overflow raises AFTER the
    capacity was grown and leaves the later frames pending (ADVICE r1); the Gaussian capacity of the sharded forward is learnt from
    status word 4; a barrier timeout is an error; freeze() drains and stops tracking."""
    cap = sgb.InstanceCapacity(headroom=1.25)
    cap.observe(10_000)
    cap.track(_status(9_000, n_sel=2_000), _FakeEvent())
    late = _FakeEvent(done=False)
    cap.track(_status(8_000, n_sel=2_100), late)
    cap.check()                                    # first frame consumed, second not arrived yet
    assert cap.gaussian_capacity == int(2_000 * 1.25) + 1024 and len(cap._pending) == 1 and not late.waited
    cap.check(wait=True)
    assert late.waited and cap.gaussian_capacity == int(2_100 * 1.25) + 1024 and not cap._pending
    assert len(cap._pool) == 2                      # the pinned words are recycled
    # overflow of the instance capacity, then of the Gaussian capacity: each reported once, in order, capacity grown first
    cap.track(_status(50_000, overflow=1, n_sel=2_000), _FakeEvent())
    cap.track(_status(9_000, overflow=2, n_sel=9_000), _FakeEvent())
    with pytest.raises(_capi.SgrError, match="instance capacity .* overflowed .*50000"):
        cap.check()
    assert cap.capacity == int(50_000 * 1.25) + 4096 and len(cap._pending) == 1
    with pytest.raises(_capi.SgrError, match="Gaussian capacity .* overflowed .*9000"):
        cap.check()
    assert cap.gaussian_capacity == int(9_000 * 1.25) + 1024 and not cap._pending
    cap.track(_status(100, timed_out=7), _FakeEvent())
    with pytest.raises(_capi.SgrError, match="barrier of epoch 7 timed out"):
        cap.check()
    ev = _FakeEvent(done=False)
    cap.track(_status(100), ev)
    assert cap.freeze().frozen and ev.waited and not cap._pending    # freeze() drains what is in flight first
    assert not cap.freeze(False).frozen


def test_header_compiles_as_c_and_struct_layouts_match_ctypes(tmp_path):
    """include/sgr.h is a plain-C header (no C++, no torch types) and EVERY ctypes mirror in _capi.py has the same size and
    field offsets as its C struct — the boundary a cgo / JNI / ctypes binding would be written against."""
    import subprocess
    src = tmp_path / "layout.c"
    structs = ["SgrFrame", "SgrPeers", "SgrSegment", "SgrSegmentGrads", "SgrStatSegment", "SgrAdamTensor", "SgrStateLayout"]
    status = ["INSTANCES", "OVERFLOW", "EMITTED", "NEAR", "NEAR_END", "SPLIT_K", "SPLIT_FIT", "FAR_END"]
    body = ['#include <stdio.h>', '#include <stddef.h>', '#include "sgr.h"', 'int main(void) {']
    for name in structs:
        body.append(f'  printf("{name} %zu\\n", sizeof({name}));')
        body += [f'  printf("{name}.{f[0]} %zu\\n", offsetof({name}, {f[0]}));' for f in getattr(_capi, name)._fields_]
    body += ['  printf("SGR_MAX_PEERS %d\\n", SGR_MAX_PEERS);', '  printf("SGR_ABI_VERSION %d\\n", SGR_ABI_VERSION);',
             '  printf("SGR_MAX_FOURIER %d\\n", SGR_MAX_FOURIER);']
    body += [f'  printf("SGR_STATUS_{w} %d\\n", SGR_STATUS_{w});' for w in status] + ['  return 0;', '}']
    src.write_text("\n".join(body))
    exe = tmp_path / "layout"
    subprocess.run(["/usr/bin/gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    out = dict(line.rsplit(" ", 1) for line in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines())
    for name in structs:
        ct = getattr(_capi, name)
        assert int(out[name]) == C.sizeof(ct), name
        for f in ct._fields_:
            assert int(out[f"{name}.{f[0]}"]) == getattr(ct, f[0]).offset, (name, f[0])
    assert int(out["SGR_MAX_PEERS"]) == _capi.MAX_PEERS and int(out["SGR_ABI_VERSION"]) == _capi.ABI_VERSION
    assert int(out["SGR_MAX_FOURIER"]) == _capi.MAX_FOURIER
    for w in status:
        assert int(out[f"SGR_STATUS_{w}"]) == getattr(_capi, f"STATUS_{w}"), w


def test_gaussian_sharded_entry_points_validate_before_touching_cuda():
    """Argument errors of the multi-GPU entry points come back as SGR_EINVAL with a message — no CUDA call is made, so
    this runs without a GPU."""
    L = _capi.lib()
    assert L.sgr_record_bytes() == 48
    fr = _capi.SgrFrame()
    fr.P, fr.width, fr.height, fr.D, fr.M = 100, 64, 64, 0, 0
    fr.tan_fovx, fr.tan_fovy, fr.scale_modifier = 0.5, 0.5, 1.0
    err = lambda: L.sgr_last_error().decode()
    # sgr_project: camera pointers are checked first
    assert L.sgr_project(C.byref(fr), None, None, None, None, None, None, None, None, None, None) == -1 and "camera" in err()
    # sgr_forward_records: outputs, then radii
    assert L.sgr_forward_records(C.byref(fr), None, None, None, None, None, None, None, 0, None, 0, _capi.ALLOC_FN(), None, None, None,
                                 None, 0, -1, None) == -1 and "output image" in err()
    # peer table validation
    assert L.sgr_scatter_records(C.byref(fr), None, None, None, None) == -1 and "peers is NULL" in err()
    pe = _capi.SgrPeers()
    pe.world, pe.rank, pe.chunk = 0, 0, 100
    assert L.sgr_scatter_records(C.byref(fr), C.byref(pe), None, None, None) == -1 and "bad peer table" in err()
    pe.world = _capi.MAX_PEERS + 1
    assert L.sgr_gather_grad2d(C.byref(fr), C.byref(pe), None, None, None, None) == -1 and "bad peer table" in err()
    pe.world, pe.rank, pe.chunk = 2, 1, 50
    assert L.sgr_scatter_records(C.byref(fr), C.byref(pe), None, None, None) == -1 and "smaller than the local" in err()
    pe.chunk = 100
    assert L.sgr_scatter_records(C.byref(fr), C.byref(pe), None, None, None) == -1 and "entry 0 is NULL" in err()


def test_sh_degree_and_alignment_validated_before_touching_cuda():
    """An active SH degree with more coefficients than stored (the kernels would evaluate uninitialised ones), and rotation / SH
    rows or their gradients off 16-byte alignment (16-byte vector loads and stores would fault), come back as SGR_EINVAL from
    every entry point that takes them.  The pointers are never dereferenced: validation precedes any CUDA call."""
    L = _capi.lib()
    err = lambda: L.sgr_last_error().decode()
    ok, off = C.c_void_p(1 << 20), C.c_void_p((1 << 20) + 4)  # 16-byte aligned, one float past it
    fr = _capi.SgrFrame()
    fr.P, fr.width, fr.height, fr.D, fr.M = 100, 64, 64, 1, 16
    fr.tan_fovx, fr.tan_fovy, fr.scale_modifier = 0.5, 0.5, 1.0
    fr.bg = fr.viewmatrix = fr.projmatrix = fr.campos = ok.value

    def project(shs, rot):
        return L.sgr_project(C.byref(fr), ok, shs, None, ok, ok, rot, None, ok, ok, None)

    for D, M in ((3, 9), (2, 4), (1, 1), (3, 15)):
        fr.D, fr.M = D, M
        assert project(ok, ok) == -1 and "SH degree" in err(), (D, M)
    fr.D, fr.M = 1, 16
    assert project(off, ok) == -1 and "shs is not 16-byte aligned" in err()
    assert project(ok, off) == -1 and "rotations is not 16-byte aligned" in err()
    for M in (4, 9, 25):  # whatever the row width: the staged and unstaged paths read rotations as float4 too
        fr.M = M
        assert project(ok, off) == -1 and "rotations" in err(), M
    fr.M = 16
    assert L.sgr_forward_bounded(C.byref(fr), ok, ok, None, None, ok, ok, off, None, ok, ok, ok, None, ok, ok, 1 << 30, ok, 1 << 30,
                                 ok, 1 << 30, 0, None) == -1 and "rotations" in err()
    assert L.sgr_visible_filter(C.byref(fr), ok, ok, off, None, ok, ok, None) == -1 and "rotations" in err()

    def backward(shs, rot, dsh, drot, D=1, M=16):
        fr.D, fr.M = D, M
        return L.sgr_backward_geom(C.byref(fr), ok, shs, None, ok, rot, None, ok, ok, ok, ok, ok, dsh, None, ok, ok, drot, None, None)

    assert backward(ok, ok, ok, ok, D=3, M=9) == -1 and "SH degree" in err()
    for args, what in (((off, ok, ok, ok), "shs"), ((ok, off, ok, ok), "rotations"), ((ok, ok, off, ok), "dL_dsh"),
                       ((ok, ok, ok, off), "dL_drotations")):
        assert backward(*args) == -1 and f"{what} is not 16-byte aligned" in err(), what


def test_peer_workspace_layout_is_aligned_and_ordered():
    from street_gaussians_b200.sharded import PeerWorkspace
    st = sgb.GaussianRasterizationSettings(480, 640, 0.5, 0.4, torch.zeros(3), 1.0, torch.eye(4), torch.eye(4), 3, torch.zeros(3), False, False)
    P_total = 8 * 12_501
    gb, ib, off_radii, off_grad, off_flags, total = PeerWorkspace.layout(st, P_total, torch.device("cpu"))
    assert gb >= P_total * 48 and off_radii >= gb and off_radii % 256 == 0
    assert off_grad >= off_radii + 4 * P_total and off_grad % 256 == 0 and ib > 0
    assert off_flags >= off_grad + 48 * P_total and off_flags % 256 == 0 and total == off_flags + 256  # barrier pad: 16 x u32, padded


def test_peer_workspace_emulation_wires_the_peer_table():
    """PeerWorkspace.emulate on CPU buffers: every rank's SgrPeers points at every buffer with the same section offsets,
    and the torch views (gathered records inside geom, radii_all, grad2d) sit at those offsets."""
    from street_gaussians_b200.sharded import PeerWorkspace
    st = sgb.GaussianRasterizationSettings(96, 128, 0.5, 0.4, torch.zeros(3), 1.0, torch.eye(4), torch.eye(4), 0, torch.zeros(3), False, False)
    world, chunk = 3, 11
    wss = PeerWorkspace.emulate(st, chunk, world, torch.device("cpu"))
    bases = [ws.buf.data_ptr() for ws in wss]
    for r, ws in enumerate(wss):
        assert (ws.peers.world, ws.peers.rank, ws.peers.chunk) == (world, r, chunk) and ws.P_total == world * chunk and not ws.in_flight
        assert ws.geom.data_ptr() == bases[r] and ws.radii_all.data_ptr() == bases[r] + ws.off_radii
        assert ws.grad2d.data_ptr() == bases[r] + ws.off_grad and ws.grad2d.shape == (world * chunk, 12)
        assert ws.radii_all.dtype == torch.int32 and ws.radii_all.shape == (world * chunk,)
        for p in range(world):
            assert ws.peers.records[p] == bases[p] and ws.peers.radii[p] == bases[p] + ws.off_radii
            assert ws.peers.grad2d[p] == bases[p] + ws.off_grad and ws.peers.flags[p] == bases[p] + ws.off_flags
        assert int(ws.buf[ws.off_flags:].sum()) == 0 and ws.epoch == 0  # barrier pads start at epoch 0
        assert ws.next_epochs(2) == 2 and ws.next_epochs() == 3
        ws.barrier()  # no symmetric-memory handle in emulation: a no-op
