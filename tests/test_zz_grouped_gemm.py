"""Grouped wgmma GEMMs: linears that share their input (q/k/v, gate/up) as ONE forward or transposed launch over the
row-concatenated weight, at prefill batches and in the backward, for every scheme the GEMM covers.

Results are checked bit-exactly on the integer lattice of test_zz_gemm_exact.py.  A group case draws ONE lattice case
for the concatenated rows (so scales, and the bounds that make every sum exact, are those of the whole group) and gives
every segment its own codebooks; the exact result of the group is the segments' exact results, concatenated (forward)
or summed (transposed).  Runs after test_zz_gemm_exact.py (`zz`): forced-plan cases set AQLM_B200_* switches and
restore them on the way out.
"""
import ctypes
import math
import os
import sys

import numpy as np
import pytest
import torch
from helpers import TOL_NORTH_STAR, make_module, to_torch
from test_zz_gemm_exact import (DEV, DT_ID, DTYPES, GEMM_SCHEMES, WS_COUNTERS, _assert_tickets_clean, assert_exact,
                                exact_forward, exact_transposed, expected_ws, lattice_case, lattice_go, n_tile_of,
                                round_to, seed_of, tunables)
from test_zz_sharded_prefill import _descriptor, _free_port

from oracle import aqlm_oracle as O

gpu = pytest.mark.gpu

GROUP_IN = 1152                                     # 18 k-blocks; 16-byte code rows for every scheme, 1x8 included
SEGMENTS = [[200, 72, 56], [128, 128], [256]]       # segment ends inside a 128-row tile, on a tile edge, one segment
BATCHES = [9, 64, 300]


# ---- group cases ----------------------------------------------------------------------------------------------------
def group_case(seed, fin, segs, K, nbits, batch, dtype=torch.float16, bias=True, unit_scales=False):
    """One lattice case over sum(segs) rows (codes, scales, bias, x) with fresh codebooks per segment.  Returns the
    per-segment cases (numpy, for the exact references) and the fused device tensors a group holds."""
    base = lattice_case(seed, fin, sum(segs), K, nbits, batch=batch, bias=bias, dtype=dtype, unit_scales=unit_scales)
    cases, off = [], 0
    for i, n in enumerate(segs):
        cb = lattice_case(seed_of("cb", seed, i), fin, n, K, nbits, dtype=dtype)["codebooks"]
        cases.append(dict(x=base["x"], codes=base["codes"][off:off + n], codebooks=cb, scales=base["scales"][off:off + n],
                          bias=None if base["bias"] is None else base["bias"][off:off + n]))
        off += n
    ts = [to_torch(c, DEV, dtype) for c in cases]
    fused = dict(x=ts[0]["x"], codes=torch.cat([t["codes"] for t in ts]).contiguous(),
                 codebooks=torch.stack([t["codebooks"] for t in ts]).contiguous(),
                 scales=torch.cat([t["scales"] for t in ts]).contiguous(),
                 bias=torch.cat([t["bias"] for t in ts]).contiguous() if bias else None)
    return cases, fused


def exact_group_forward(cases, partial=False):
    if partial:
        return np.concatenate([O.dequantize_gemm(c["x"], c["codes"], c["codebooks"], None, None, dtype=np.float64)
                               for c in cases], axis=1)
    return np.concatenate([exact_forward(c) for c in cases], axis=1)


def exact_group_transposed(cases, go):
    off, acc = 0, 0
    for c in cases:
        n = c["codes"].shape[0]
        acc = acc + exact_transposed(c, go[:, off:off + n])
        off += n
    return acc


def _group_weight(f, scales=True, bias=True):
    from aqlm_b200.inference_kernels import cuda_kernel

    return cuda_kernel.make_weight(f["codes"], f["codebooks"][0], f["scales"].reshape(-1) if scales else None,
                                   f["bias"] if bias else None)


def _run_grouped(f, segs, batch, partial=False):
    """matmat_dequant_grouped; returns (y as numpy, workspace bytes of the concatenated descriptor, launches)."""
    from aqlm_b200 import _cabi
    from aqlm_b200.inference_kernels import cuda_kernel

    need = _cabi.lib().aqlm_b200_matmat_dequant_workspace_bytes(ctypes.byref(_group_weight(f)), batch)
    before = _cabi.launch_count()
    y = cuda_kernel.matmat_dequant_grouped(f["x"], f["codes"], f["codebooks"], f["scales"], f["bias"], segs,
                                           partial=partial)
    launches = _cabi.launch_count() - before
    assert y is not None, "the grouped GEMM refused a layout it covers"
    assert y.dtype == (torch.float32 if partial else f["x"].dtype) and y.shape == (batch, sum(segs))
    if need:
        _assert_tickets_clean("grouped forward")
    return y.float().cpu().numpy(), need, launches


def _run_grouped_t(f, segs, go):
    from aqlm_b200 import _cabi
    from aqlm_b200.inference_kernels import cuda_kernel

    batch = go.shape[0]
    need = _cabi.lib().aqlm_b200_matmat_dequant_transposed_workspace_bytes(ctypes.byref(_group_weight(f, bias=False)),
                                                                           batch)
    before = _cabi.launch_count()
    gx = cuda_kernel.matmat_dequant_transposed_grouped(go, f["codes"], f["codebooks"], f["scales"], segs)
    launches = _cabi.launch_count() - before
    assert gx is not None, "the grouped transposed GEMM refused a layout it covers"
    if need:
        _assert_tickets_clean("grouped transposed")
    return gx.float().cpu().numpy(), need, launches


def _seg_id(segs):
    return "seg" + "-".join(map(str, segs))


# ==== CPU: argument checks without a device ==========================================================================
def _call(L, transposed, w, seg, n_seg, b=16, y=16, batch=64):
    seg_arr = None if seg is None else (ctypes.c_int64 * max(len(seg), 1))(*seg)
    if transposed:
        return L.aqlm_b200_matmat_dequant_transposed_grouped(ctypes.byref(w), seg_arr, n_seg, b, y, batch, None, 0, None)
    return L.aqlm_b200_matmat_dequant_grouped(ctypes.byref(w), seg_arr, n_seg, b, y, batch, 0, None, 0, None)


@pytest.mark.parametrize("transposed", [False, True], ids=["forward", "transposed"])
def test_grouped_argument_checks_without_a_device(transposed):
    from aqlm_b200 import _cabi

    L = _cabi.lib()
    S, U = _cabi.ERR_SHAPE, _cabi.ERR_UNSUPPORTED
    w = _descriptor()  # 1024 -> 256, 1x16, in_group 8
    assert _call(L, transposed, w, [64, 64, 64, 64], 0) == S
    assert _call(L, transposed, w, [64, 64, 64, 32, 32], 5) == S
    assert b"1..4 segments" in L.aqlm_b200_last_error()
    assert _call(L, transposed, w, None, 1) == S
    assert _call(L, transposed, w, [128, 64], 2) == S            # 192 rows, not 256
    assert b"add up" in L.aqlm_b200_last_error()
    assert _call(L, transposed, w, [256, 0], 2) == S             # an empty segment
    assert _call(L, transposed, w, [300, -44], 2) == S           # a negative one that makes the sum right
    assert _call(L, transposed, w, [256], 1, b=None) == S
    assert _call(L, transposed, w, [256], 1, batch=-1) == S
    # layouts the wgmma kernels do not take: ERR_UNSUPPORTED with a message, never a GEMV fallback
    for kw in (dict(in_group_size=16), dict(num_codebooks=3, nbits_per_codebook=8), dict(nbits_per_codebook=12)):
        assert _call(L, transposed, _descriptor(**kw), [128, 128], 2) == U, kw
        assert b"grouped" in L.aqlm_b200_last_error()
    assert _call(L, transposed, _descriptor(), [128, 128], 2, b=24) == U   # input / grad_output not 16-byte aligned
    assert _call(L, transposed, _descriptor(codes=24), [128, 128], 2) == U
    if transposed:  # out_features % 8 != 0 (the forward takes it)
        assert _call(L, transposed, _descriptor(out_features=252), [126, 126], 2) == U
        assert b"% 8" in L.aqlm_b200_last_error()
    else:           # in_features % 64 != 0, with 16-byte code rows (4x8: 528 bytes): only the k-block rules it out
        assert _call(L, transposed, _descriptor(in_features=1056, num_codebooks=4, nbits_per_codebook=8), [128, 128],
                     2) == U
        assert b"% 64" in L.aqlm_b200_last_error()
    assert _call(L, transposed, w, [128, 128], 2, batch=0) == _cabi.OK   # nothing to do: no device needed
    if torch.cuda.is_available():
        return  # the calls below would launch on the dummy pointers
    for ok_shape in ([256], [200, 56], [64, 64, 64, 64]):
        assert _call(L, transposed, w, ok_shape, len(ok_shape)) in (_cabi.ERR_CUDA, _cabi.ERR_ARCH)


def test_partial_flag_needs_no_scales_without_a_device():
    from aqlm_b200 import _cabi

    L = _cabi.lib()
    w = _descriptor()
    w.scales = None
    seg = (ctypes.c_int64 * 2)(128, 128)
    assert L.aqlm_b200_matmat_dequant_grouped(ctypes.byref(w), seg, 2, 16, 16, 64, 0, None, 0, None) == _cabi.ERR_SHAPE
    assert b"scales" in L.aqlm_b200_last_error()
    assert L.aqlm_b200_matmat_dequant_transposed_grouped(ctypes.byref(w), seg, 2, 16, 16, 64, None, 0,
                                                         None) == _cabi.ERR_SHAPE
    if torch.cuda.is_available():
        return
    rc = L.aqlm_b200_matmat_dequant_grouped(ctypes.byref(w), seg, 2, 16, 16, 64, _cabi.FLAG_PARTIAL_F32, None, 0, None)
    assert rc in (_cabi.ERR_CUDA, _cabi.ERR_ARCH), rc


def test_storage_fusion_follows_the_gemm_schemes():
    """The group fuses storage for exactly the schemes the grouped GEMM takes (checked on meta tensors: no device)."""
    import aqlm_b200
    from aqlm_b200.grouped import _check_members, gemm_scheme

    def linear(K, nbits, g, out=64):
        return aqlm_b200.QuantizedLinear(256, out, g, 1, K, nbits, bias=False, device="meta", dtype=torch.float16)

    for K, nbits in GEMM_SCHEMES:
        assert gemm_scheme(linear(K, nbits, 8))
    for K, nbits, g in [(1, 16, 16), (3, 8, 8), (2, 12, 8), (16, 8, 8)]:
        assert not gemm_scheme(linear(K, nbits, g))
        assert not _check_members([linear(K, nbits, g), linear(K, nbits, g)])
    assert not _check_members([linear(2, 8, 8)] * 2)  # meta, not CUDA: nothing to launch on
    with pytest.raises(ValueError):
        _check_members([linear(2, 8, 8), linear(1, 8, 8)])


# ==== GPU: forward ===================================================================================================
def _fwd_cases():
    return [pytest.param(K, nbits, dtype, batch, segs, id=f"{K}x{nbits}-{DT_ID[dtype]}-bs{batch}-{_seg_id(segs)}")
            for K, nbits in GEMM_SCHEMES for dtype in DTYPES for batch in BATCHES for segs in SEGMENTS]


@gpu
@pytest.mark.parametrize("K,nbits,dtype,batch,segs", _fwd_cases())
def test_grouped_forward_exact(K, nbits, dtype, batch, segs):
    cases, f = group_case(seed_of("gfwd", K, nbits, batch, segs), GROUP_IN, segs, K, nbits, batch, dtype)
    y, need, launches = _run_grouped(f, segs, batch)
    assert launches == 1, "a group is ONE wgmma GEMM launch"
    assert_exact(y, round_to(exact_group_forward(cases), dtype), f"grouped {K}x{nbits} {segs} bs={batch}",
                 n_tile=n_tile_of(batch))


FORCED = [(tm, ks) for tm in (127, 40) for ks in (1, 3, 16)]


@gpu
@pytest.mark.parametrize("K,nbits", [(1, 16), (2, 8), (8, 8), (4, 16)])
@pytest.mark.parametrize("tile_m,ksplit", FORCED, ids=[f"tm{tm}-ks{ks}" for tm, ks in FORCED])
def test_grouped_forward_forced_plan_exact(K, nbits, tile_m, ksplit):
    """Tiles of 127 and 40 rows straddle the segment ends 200 and 272; the split count shows in the workspace the
    concatenated descriptor asks for."""
    segs, batch = [200, 72, 56], 64 if ksplit != 16 else 300
    dtype = DTYPES[(tile_m + ksplit) % 2]
    cases, f = group_case(seed_of("gforced", K, nbits, tile_m, ksplit), GROUP_IN, segs, K, nbits, batch, dtype)
    with tunables(gemm_tile_m=tile_m, gemm_ksplit=ksplit):
        y, need, launches = _run_grouped(f, segs, batch)
    assert launches == 1
    assert need == expected_ws(math.ceil(sum(segs) / tile_m), batch, min(ksplit, GROUP_IN // 64)), need
    assert_exact(y, round_to(exact_group_forward(cases), dtype), f"grouped {K}x{nbits} tile_m={tile_m} ksplit={ksplit}",
                 tile_m=tile_m, n_tile=n_tile_of(batch))


@gpu
def test_grouped_workspace_is_the_concatenated_query():
    """The workspace the ungrouped query gives for the concatenated descriptor is exactly what the grouped call uses:
    with that many bytes the split plan runs (partials written), with one byte less it runs unsplit (untouched)."""
    from aqlm_b200 import _cabi

    L = _cabi.lib()
    segs, batch, dtype = [200, 72, 56], 64, torch.float16
    cases, f = group_case(seed_of("gws"), GROUP_IN, segs, 1, 16, batch, dtype)
    ref = round_to(exact_group_forward(cases), dtype)
    w = _group_weight(f)
    seg = (ctypes.c_int64 * 3)(*segs)
    out = torch.empty((batch, sum(segs)), dtype=dtype, device=DEV)
    st = torch.cuda.current_stream().cuda_stream
    with tunables(gemm_ksplit=5):
        need = L.aqlm_b200_matmat_dequant_workspace_bytes(ctypes.byref(w), batch)
        assert need > WS_COUNTERS
        for nbytes, split in ((need, True), (need - 1, False)):
            ws = torch.zeros(need, dtype=torch.uint8, device=DEV)
            ws[WS_COUNTERS:] = 0xA5
            out.fill_(float("nan"))
            _cabi.check(L.aqlm_b200_matmat_dequant_grouped(ctypes.byref(w), seg, 3, f["x"].data_ptr(), out.data_ptr(),
                                                           batch, 0, ws.data_ptr(), nbytes, st))
            torch.cuda.synchronize()
            assert_exact(out.float().cpu().numpy(), ref, f"grouped, workspace of {nbytes} bytes")
            assert int(torch.count_nonzero(ws[:WS_COUNTERS])) == 0
            assert bool((ws[WS_COUNTERS:] == 0xA5).all()) != split, (nbytes, split)


# ==== GPU: other entry paths =========================================================================================
@gpu
@pytest.mark.parametrize("K,nbits", [(1, 16), (2, 8), (8, 16)])
@pytest.mark.parametrize("batch", [9, 300])
def test_grouped_partial_f32_without_scales_exact(K, nbits, batch):
    from aqlm_b200 import _cabi
    from aqlm_b200.inference_kernels import cuda_kernel

    segs = [200, 72, 56]
    cases, f = group_case(seed_of("gpartial", K, nbits, batch), GROUP_IN, segs, K, nbits, batch, bias=False)
    before = _cabi.launch_count()
    # the flagged call reads neither scales nor bias: NULL for both
    p = cuda_kernel.matmat_dequant_grouped(f["x"], f["codes"], f["codebooks"], None, None, segs, partial=True)
    assert _cabi.launch_count() - before == 1
    assert p.dtype == torch.float32
    assert_exact(p.cpu().numpy(), exact_group_forward(cases, partial=True), f"grouped partial {K}x{nbits} bs={batch}",
                 n_tile=n_tile_of(batch))


T_FORCED = [(1, 16, None), (1, 16, 3), (8, 8, 16), (2, 16, 5)]


@gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("K,nbits,ksplit", T_FORCED, ids=[f"{k}x{n}-ks{s}" for k, n, s in T_FORCED])
@pytest.mark.parametrize("batch", [9, 64, 300])
def test_grouped_transposed_exact(K, nbits, ksplit, dtype, batch):
    """grad_in = sum over segments of (grad_out_i * scales_i) . W_i, each segment with its own scales and codebooks."""
    segs = [200, 72, 56]  # 328 out rows: 6 k-blocks, segment ends inside k-blocks 3 and 4
    cases, f = group_case(seed_of("gt", K, nbits, ksplit, batch), GROUP_IN, segs, K, nbits, 1, dtype, bias=False)
    go = lattice_go(seed_of("gt-go", K, nbits, ksplit, batch), batch, sum(segs))
    with tunables(gemm_ksplit=ksplit):
        gx, need, launches = _run_grouped_t(f, segs, torch.from_numpy(go).to(dtype).to(DEV))
    assert launches == 1
    if ksplit is not None:
        assert need == expected_ws(math.ceil(GROUP_IN / 128), batch, min(ksplit, math.ceil(sum(segs) / 64))), need
    assert_exact(gx, round_to(exact_group_transposed(cases, go), dtype), f"grouped transposed {K}x{nbits} bs={batch}",
                 n_tile=n_tile_of(batch))


@gpu
@pytest.mark.parametrize("batch", [16, 300])
def test_unsupported_layouts_return_none_and_the_group_runs_its_members(batch):
    """in_group 16 and in_features % 64 != 0: the grouped GEMMs answer ERR_UNSUPPORTED (None in Python) and the group's
    output is its members' output, exactly."""
    from aqlm_b200.grouped import QuantizedLinearGroup
    from aqlm_b200.inference_kernels import cuda_kernel

    segs = [128, 64, 64]
    for K, nbits, g, fin in [(1, 16, 16, 1024), (2, 8, 8, 1096)]:
        base = lattice_case(seed_of("gunsup", g, fin, batch), fin, sum(segs), K, nbits, g, batch=batch)
        t = to_torch(base, DEV)
        cb = torch.stack([t["codebooks"]] * len(segs)).contiguous()
        assert cuda_kernel.matmat_dequant_grouped(t["x"], t["codes"], cb, t["scales"], t["bias"], segs) is None
        go = torch.ones((batch, sum(segs)), dtype=torch.float16, device=DEV)
        assert cuda_kernel.matmat_dequant_transposed_grouped(go, t["codes"], cb, t["scales"], segs) is None
        layers, off = [], 0
        for n in segs:
            sub = dict(base, codes=base["codes"][off:off + n], scales=base["scales"][off:off + n], bias=base["bias"][off:off + n])
            layers.append(make_module(sub, DEV)[0])
            off += n
        grp = QuantizedLinearGroup(layers)
        assert grp.fused == (g == 8)
        with torch.no_grad():
            ys = grp(t["x"])
        y = torch.cat(ys, dim=-1).float().cpu().numpy()
        assert_exact(y, round_to(exact_forward(base), torch.float16), f"members of an unsupported group g={g} in={fin}")


# ==== GPU: modules ===================================================================================================
def _group_modules(cases, dtype=torch.float16):
    from aqlm_b200.grouped import QuantizedLinearGroup

    layers = [make_module(c, DEV, dtype)[0] for c in cases]
    return QuantizedLinearGroup(layers), layers


@gpu
@pytest.mark.parametrize("batch", [16, 300])
@pytest.mark.parametrize("K,nbits", [(1, 16), (2, 8)])
def test_group_module_prefill_one_launch_exact(K, nbits, batch):
    from aqlm_b200 import _cabi

    segs = [256, 128, 128]
    cases, _ = group_case(seed_of("gmod", K, nbits, batch), GROUP_IN, segs, K, nbits, batch)
    grp, _ = _group_modules(cases)
    assert grp.fused
    x = to_torch(cases[0], DEV)["x"].reshape(batch // 4 if batch % 4 == 0 else 1, -1, GROUP_IN)
    with torch.no_grad():
        grp(x)
        torch.cuda.synchronize()
        before = _cabi.launch_count()
        ys = grp(x)
        assert _cabi.launch_count() - before == 1
    assert [tuple(y.shape) for y in ys] == [tuple(x.shape[:-1]) + (n,) for n in segs]
    y = torch.cat(ys, dim=-1).reshape(batch, -1).float().cpu().numpy()
    assert_exact(y, round_to(exact_group_forward(cases), torch.float16), f"group module {K}x{nbits} bs={batch}")


@gpu
@pytest.mark.parametrize("batch", [4, 16, 300])
@pytest.mark.parametrize("K,nbits", [(1, 16), (2, 8)])
def test_group_module_input_gradient(K, nbits, batch):
    """With x.requires_grad the group runs one forward and one transposed launch; the input gradient equals the members'
    path (each member's own forward and backward, summed by autograd) and the exact one.  Unit scales and integer
    gradients keep every value, member sums included, exact in fp16."""
    from aqlm_b200 import _cabi

    segs = [128, 64, 64]
    cases, _ = group_case(seed_of("ggrad", K, nbits, batch), GROUP_IN, segs, K, nbits, batch, unit_scales=True)
    go_np = lattice_go(seed_of("ggrad-go", batch), batch, sum(segs), x_max=1)
    go = torch.from_numpy(go_np).half().to(DEV)
    grp, _ = _group_modules(cases)
    solo = [make_module(c, DEV)[0] for c in cases]  # the same weights, not grouped
    x0 = to_torch(cases[0], DEV)["x"]

    x = x0.clone().requires_grad_(True)
    before = _cabi.launch_count()
    ys = grp(x)
    assert _cabi.launch_count() - before == 1, "one grouped forward launch"
    assert all(y.requires_grad for y in ys)
    before = _cabi.launch_count()
    torch.autograd.backward(ys, list(torch.split(go, segs, dim=-1)))
    assert _cabi.launch_count() - before == 1, "one grouped transposed launch"

    xm = x0.clone().requires_grad_(True)
    ym = [m(xm) for m in solo]
    torch.autograd.backward(ym, list(torch.split(go, segs, dim=-1)))
    for a, b in zip(ys, ym):
        assert torch.equal(a.detach(), b.detach())
    ref = exact_group_transposed(cases, go_np)
    assert_exact(x.grad.float().cpu().numpy(), round_to(ref, torch.float16), f"group input grad {K}x{nbits} bs={batch}")
    assert torch.equal(x.grad, xm.grad)


@gpu
def test_group_decode_gradient_with_unaligned_input_runs_the_members():
    """Up to 8 rows of a 1x16 group with an input that needs a gradient: an input the grouped GEMV refuses (not 16-byte
    aligned) goes through the members, and both the output and the input gradient are exact."""
    from aqlm_b200 import _cabi

    segs, batch = [128, 64, 64], 4
    cases, _ = group_case(seed_of("gunaligned"), GROUP_IN, segs, 1, 16, batch, unit_scales=True)
    grp, _ = _group_modules(cases)
    x0 = to_torch(cases[0], DEV)["x"]
    buf = torch.empty(x0.numel() + 1, dtype=x0.dtype, device=DEV)
    buf[1:].copy_(x0.reshape(-1))
    x = buf[1:].view(batch, GROUP_IN).detach().requires_grad_(True)
    assert x.data_ptr() % 16 != 0
    before = _cabi.launch_count()
    ys = grp(x)
    assert _cabi.launch_count() - before == len(segs), "one launch per member"
    assert_exact(torch.cat([y.detach() for y in ys], -1).float().cpu().numpy(),
                 round_to(exact_group_forward(cases), torch.float16), "unaligned decode through the members")
    go_np = lattice_go(seed_of("gunaligned-go"), batch, sum(segs), x_max=1)
    torch.autograd.backward(ys, list(torch.split(torch.from_numpy(go_np).half().to(DEV), segs, dim=-1)))
    assert_exact(x.grad.float().cpu().numpy(), round_to(exact_group_transposed(cases, go_np), torch.float16),
                 "unaligned decode input gradient")


@gpu
def test_group_2x8_fused_storage_prefill_and_decode():
    """A 2x8 group fuses its storage; prefill is one exact grouped GEMM, decode (<= 8 rows) runs the members' own kernels on
    views of the fused storage."""
    from aqlm_b200 import _cabi

    segs = [256, 64, 64]
    cases, _ = group_case(seed_of("g2x8"), GROUP_IN, segs, 2, 8, 64)
    grp, layers = _group_modules(cases)
    assert grp.fused
    off = 0
    for i, (m, n) in enumerate(zip(layers, segs)):
        assert m.codes.data_ptr() == grp._fused_codes[off:off + n].data_ptr()
        assert m.codebooks.data_ptr() == grp._fused_codebooks[i].data_ptr()
        off += n
    x = to_torch(cases[0], DEV)["x"]
    with torch.no_grad():
        before = _cabi.launch_count()
        ys = grp(x)
        assert _cabi.launch_count() - before == 1
        assert_exact(torch.cat(ys, -1).float().cpu().numpy(), round_to(exact_group_forward(cases), torch.float16),
                     "2x8 group prefill")
        before = _cabi.launch_count()
        yd = grp(x[:4])
        assert _cabi.launch_count() - before == len(segs), "decode: one launch per member"
    ref4 = round_to(np.concatenate([exact_forward(c, x=c["x"][:4]) for c in cases], axis=1), torch.float16)
    assert_exact(torch.cat(yd, -1).float().cpu().numpy(), ref4, "2x8 group decode through the members")


@pytest.fixture
def aqlm_hf(monkeypatch):
    """`aqlm` resolves to this package and Hugging Face's AQLM quantizer skips its `accelerate` check (as in
    test_checkpoint.py)."""
    pytest.importorskip("transformers")
    import aqlm_b200

    saved = {k: v for k, v in sys.modules.items() if k == "aqlm" or k.startswith("aqlm.")}
    aqlm_b200.install_as_aqlm()
    import transformers.quantizers.quantizer_aqlm as QA

    monkeypatch.setattr(QA, "is_accelerate_available", lambda: True)
    yield aqlm_b200
    for k in [k for k in sys.modules if k == "aqlm" or k.startswith("aqlm.")]:
        del sys.modules[k]
    sys.modules.update(saved)


@gpu
@pytest.mark.parametrize("K,nbits", [(1, 16), (2, 8)])
def test_checkpoint_prefill_with_grouped_gemm(tmp_path, aqlm_hf, K, nbits):
    """A synthetic Llama checkpoint at 20 rows: after fuse_shared_input_linears every layer makes 3 fewer launches (q/k/v
    and gate/up are one grouped GEMM each), the logits still match the dense dequantized model, the state dict keys
    are unchanged."""
    from test_checkpoint import write_synthetic_checkpoint
    from transformers import AutoModelForCausalLM, LlamaForCausalLM

    from aqlm_b200 import _cabi

    cfg, dense_sd, _ = write_synthetic_checkpoint(str(tmp_path / "m"), K, nbits, seed=5)
    model = AutoModelForCausalLM.from_pretrained(str(tmp_path / "m"), dtype=torch.float16).to(DEV).eval()
    dense = LlamaForCausalLM(cfg).half()
    dense.load_state_dict(dense_sd)
    dense = dense.to(DEV).eval()
    ids = torch.randint(0, cfg.vocab_size, (4, 5), device=DEV, generator=torch.Generator(DEV).manual_seed(1))
    names = sorted(model.state_dict().keys())
    with torch.no_grad():
        ld = dense(ids).logits.float()
        model(ids)
        c0 = _cabi.launch_count()
        plain = model(ids).logits.float()
        plain_launches = _cabi.launch_count() - c0
        assert aqlm_hf.fuse_shared_input_linears(model) == 2 * cfg.num_hidden_layers
        model(ids)
        c0 = _cabi.launch_count()
        fused = model(ids).logits.float()
        fused_launches = _cabi.launch_count() - c0
    assert fused_launches == plain_launches - 3 * cfg.num_hidden_layers, (plain_launches, fused_launches)
    for lq in (plain, fused):
        rel = ((lq - ld).abs().mean() / ld.abs().mean()).item()
        assert rel < 5e-3, rel
    assert sorted(model.state_dict().keys()) == names


@gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
def test_sharded_group_world1_prefill_exact(dtype):
    """ONE grouped GEMM launch for the group's partials and ONE scale_bias launch."""
    from aqlm_b200 import _cabi
    from aqlm_b200.grouped import ShardedQuantizedLinearGroup
    from aqlm_b200.sharded import ShardedQuantizedLinear

    segs, batch = [200, 72, 56], 64
    cases, _ = group_case(seed_of("gsharded", dtype), GROUP_IN, segs, 1, 16, batch, dtype)
    ms = []
    for c in cases:
        t = to_torch(c, DEV, dtype)
        ms.append(ShardedQuantizedLinear.from_full(t["codes"], t["codebooks"], t["scales"], t["bias"], rank=0,
                                                   world_size=1))
    grp = ShardedQuantizedLinearGroup(ms)
    assert grp.fused
    x = to_torch(cases[0], DEV, dtype)["x"]
    with torch.no_grad():
        grp(x)
        torch.cuda.synchronize()
        before = _cabi.launch_count()
        ys = grp(x)
        assert _cabi.launch_count() - before == 2
    assert_exact(torch.cat(ys, -1).float().cpu().numpy(), round_to(exact_group_forward(cases), dtype),
                 f"sharded group world 1 bs={batch}")


def _two_gpu_group_worker(rank, world, port, ret):
    import torch.distributed as dist

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("gloo", rank=rank, world_size=world)  # only used to exchange IPC handles
    try:
        from aqlm_b200 import _cabi
        from aqlm_b200.grouped import ShardedQuantizedLinearGroup
        from aqlm_b200.peer import PeerComm
        from aqlm_b200.sharded import ShardedQuantizedLinear

        dev, batch = f"cuda:{rank}", 64
        comm = PeerComm(max_elems=4 * 4096)  # batch 64 x 768 outputs: 4 exchanges of 21 rows
        cases = [O.make_case(8400 + i, 2048, o, 1, 16, 8, batch, bias=False) for i, o in enumerate((512, 128, 128))]
        for cc in cases[1:]:
            cc["x"] = cases[0]["x"]
        ms = []
        for cc in cases:
            tt = to_torch(cc, dev)
            ms.append(ShardedQuantizedLinear.from_full(tt["codes"], tt["codebooks"], tt["scales"], None, rank=rank,
                                                       world_size=world, peer_comm=comm))
        grp = ShardedQuantizedLinearGroup(ms)
        x = to_torch(cases[0], dev)["x"]
        with torch.no_grad():
            grp(x)
            torch.cuda.synchronize()
            before = _cabi.launch_count()
            ys = grp(x)
            torch.cuda.synchronize()
        launches = _cabi.launch_count() - before
        errs = []
        for cc, y in zip(cases, ys):
            layer, t = make_module(cc, dev)
            with torch.no_grad():
                ref = layer(t["x"]).float().cpu().numpy()
            errs.append(O.relative_error(y.float().cpu().numpy(), ref))
        ret[rank] = (launches, errs)
    finally:
        dist.barrier()
        dist.destroy_process_group()


@gpu
@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_sharded_group_prefill_two_gpus():
    """One grouped GEMM and one (chunked) exchange for the whole group on each rank."""
    import torch.multiprocessing as mp

    ret = mp.Manager().dict()
    mp.spawn(_two_gpu_group_worker, args=(2, _free_port(), ret), nprocs=2, join=True)
    chunks = math.ceil(64 / ((4 * 4096) // 768))
    for r in range(2):
        launches, errs = ret[r]
        assert launches == 1 + chunks, (r, launches)
        assert all(e < TOL_NORTH_STAR for e in errs), (r, errs)
