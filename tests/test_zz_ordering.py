"""Ordering and concurrency: every kernel checked bit-exactly when its operands were written by the kernel just before
it, across training steps without a host sync, on concurrent streams, beside a graph replay, from several host threads
and on a second device.

The bit-exact suites run one call at a time: one stream, weights uploaded by a host copy, a synchronize before each
check.  Real use breaks each of these:

A  With programmatic dependent launch (AQLM_B200_PDL=1, the default) the forward GEMM, the GEMV and the LUT GEMVs read
   codes, codebooks and scales in their prologue, before the dependency wait.  `optimizer.step()` rewrites codebooks,
   scales and bias in place with a kernel, and the next forward launches right behind it.  Each step here rewrites
   one operand with an in-place torch kernel that keeps it on the integer lattice of test_zz_gemm_exact.py and launches
   the op immediately after.  Every step's output is checked against the float64 model of that step's operands.
   PDL=0 is the control.
B  Training steps (forward, backward, SGD) with no host sync, against a float64 dense replica of the same steps.
C  Three streams with interleaved chains; each stream has its own workspace.
D  A CUDA-graph replay on a side stream beside eager work on the default stream, unordered against each other.
E  Host threads with their own streams launching one kernel instantiation at different shared-memory sizes.
F  Tensors on cuda:1 while cuda:0 is current.

Each scenario ends with ONE synchronize and then compares.  The CPU tests prove the scenarios have teeth: every step's
exact output differs from the previous step's in at least TEETH elements (B: the output moves by more than ten times
the tolerance), so a kernel that read the previous step's operands cannot pass.
"""
import ctypes
import math
import threading

import numpy as np
import pytest
import torch
from test_zz_gemm_exact import (B_MAX, WS_TICKETS, X_MAX, assert_exact, exact_forward, exact_transposed, lattice_bounds,
                                lattice_case, lattice_go, round_to, seed_of, tunables)
from test_zz_rounding import TEETH
from test_zz_weight_grad import E_HI, exact_weight_grad, lattice_linear

from oracle import aqlm_oracle as O

DEV = "cuda:0"
gpu = pytest.mark.gpu
F16, BF16 = torch.float16, torch.bfloat16
S = 8  # steps of scenario A: every rewrite kind at least twice


# ==== A: operands rewritten by the kernel just before ================================================================
# Rewrites, each one in-place torch kernel on the device and the same operation on the host model.  They keep every
# operand on the lattice: codebooks and activations change sign, scales halve (one exponent below the lattice's
# range; `_check_bounds` proves it exact) and double back, the bias moves to a second lattice bias and back.
REWRITES = {
    "cb.neg": ("cb", lambda t: t["cb"].neg_(), lambda v, st: -v),
    "s.half": ("s", lambda t: t["s"].mul_(0.5), lambda v, st: v * 0.5),
    "s.double": ("s", lambda t: t["s"].mul_(2), lambda v, st: v * 2),
    "b.add": ("b", lambda t: t["b"].add_(t["db"]), lambda v, st: v + st["db"]),
    "b.sub": ("b", lambda t: t["b"].sub_(t["db"]), lambda v, st: v - st["db"]),
    "x.neg": ("x", lambda t: t["x"].neg_(), lambda v, st: -v),
    "go.neg": ("go", lambda t: t["go"].neg_(), lambda v, st: -v),
    "off.add": ("off", lambda t: t["off"].add_(t["doff"]), lambda v, st: v + st["doff"]),
    "off.sub": ("off", lambda t: t["off"].sub_(t["doff"]), lambda v, st: v - st["doff"]),
}
SEQ_BIAS = ["cb.neg", "s.half", "b.add", "x.neg", "cb.neg", "s.double", "b.sub", "x.neg"]
SEQ_NO_BIAS = ["cb.neg", "s.half", "x.neg", "cb.neg", "s.double", "x.neg", "cb.neg", "s.half"]
SEQ_ROUTED = ["off.add", "cb.neg", "s.half", "x.neg", "off.sub", "cb.neg", "s.double", "x.neg"]
SEQ_WGRAD = ["cb.neg", "s.half", "x.neg", "go.neg", "cb.neg", "s.double", "x.neg", "go.neg"]

# (name, op, K, nbits, in, out, batch, dtype, switches, launches per call)
ENTRIES = [
    ("lut-cluster-2x8-bs1", "gemv", 2, 8, 1024, 200, 1, F16, {}, 1),
    ("lut-ws-8x8-bs1", "gemv", 8, 8, 1024, 200, 1, F16, {}, 1),
    ("vec-1x16-bs1", "gemv", 1, 16, 1024, 200, 1, F16, {}, 1),
    ("vec-2x8-bs5", "gemv", 2, 8, 1024, 200, 5, BF16, {}, 1),
    ("vec-1x16-bs6", "gemv", 1, 16, 1024, 200, 6, F16, {}, 1),
    ("lut-rows-2x8-bs3", "gemv", 2, 8, 1024, 200, 3, F16, {}, 3),
    ("gemm-2x8-bs17-unsplit", "gemm", 2, 8, 1152, 456, 17, F16, {"gemm_ksplit": 1}, 1),
    ("gemm-1x16-bs64-ks5", "gemm", 1, 16, 1152, 456, 64, F16, {"gemm_ksplit": 5}, 1),
    ("grouped-2x8-bs17", "grouped", 2, 8, 512, (72, 64, 64), 17, BF16, {}, 1),
    ("routed-2x8", "routed", 2, 8, 512, 136, 40, F16, {}, 1),
    ("transposed-1x16-bs64", "transposed", 1, 16, 1088, 456, 64, BF16, {}, 1),
    ("wgrad-2x8-bs64", "wgrad", 2, 8, 1152, 200, 64, F16, {}, 1),
]
ENTRY_IDS = [e[0] for e in ENTRIES]
ROUTED_E, ROUTED_OFF, ROUTED_OFF2 = 3, [0, 5, 23, 40], [0, 17, 17, 40]  # the rewrite empties expert 1


def _state(entry):
    """Host state (float32 lattice arrays, exact in fp16 and bf16) of one entry point, with its rewrite sequence."""
    name, op, K, nbits, fin, fout, batch, dtype, _, _ = entry
    rng = np.random.default_rng(seed_of("ordering", name))
    if op == "wgrad":
        lin = lattice_linear(seed_of("ordering-wgrad", name), fin, fout, K, nbits)
        # scales 2^-e with e in [0, E_HI - 1]: after `s.half` they are still on the weight-gradient lattice
        e = rng.integers(0, E_HI, size=fout)
        s = np.ldexp(np.float32(1.0), -e).astype(np.float32).reshape(fout, 1, 1, 1)
        x = rng.integers(-2, 3, size=(batch, fin)).astype(np.float32)
        go = rng.integers(-2, 3, size=(batch, fout)).astype(np.float32)
        return dict(raw=lin["raw"], codes=lin["codes"], cb=lin["codebooks"], s=s, x=x, go=go), SEQ_WGRAD
    if op in ("grouped", "routed"):
        parts = fout if op == "grouped" else [fout] * ROUTED_E
        cs = [lattice_case(seed_of("ordering", name, i), fin, o, K, nbits, batch=batch, bias=op == "grouped", dtype=dtype)
              for i, o in enumerate(parts)]
        st = dict(x=cs[0]["x"], e=(cs[0]["e_lo"], cs[0]["e_hi"]))
        if op == "grouped":
            st.update(codes=np.concatenate([c["codes"] for c in cs]), cb=np.stack([c["codebooks"] for c in cs]),
                      s=np.concatenate([c["scales"] for c in cs]), b=np.concatenate([c["bias"] for c in cs]))
            st["db"] = rng.integers(-B_MAX, B_MAX + 1, size=st["b"].shape).astype(np.float32) - st["b"]
            return st, SEQ_BIAS
        st.update(codes=np.stack([c["codes"] for c in cs]), cb=np.stack([c["codebooks"][None] for c in cs]),
                  s=np.stack([c["scales"] for c in cs]), off=np.array(ROUTED_OFF, dtype=np.int32))
        st["doff"] = np.array(ROUTED_OFF2, dtype=np.int32) - st["off"]
        return st, SEQ_ROUTED
    bias = op != "transposed"
    c = lattice_case(seed_of("ordering", name), fin, fout, K, nbits, batch=batch, bias=bias, dtype=dtype)
    st = dict(codes=c["codes"], cb=c["codebooks"], s=c["scales"], b=c["bias"], e=(c["e_lo"], c["e_hi"]),
              x=lattice_go(seed_of("ordering-go", name), batch, fout) if op == "transposed" else c["x"])
    if bias:
        st["db"] = rng.integers(-B_MAX, B_MAX + 1, size=fout).astype(np.float32) - st["b"]
        return st, SEQ_BIAS
    return st, SEQ_NO_BIAS


def _model(entry, st, rounded=True):
    """The exact output of one call on the operands in `st` (2-D, float64), rounded once to the output type; the
    weight gradient is the fp32 pair (grad_codebooks, grad_scales) flattened into one row (rounded to the parameters'
    dtype when `rounded`, as the Python op returns it)."""
    name, op, K, nbits, fin, fout, batch, dtype, _, _ = entry
    lin = lambda codes, cb, s, b=None: dict(codes=codes, codebooks=cb, scales=s, bias=b)  # noqa: E731
    if op == "wgrad":
        gcb, gs = exact_weight_grad(dict(raw=st["raw"], codebooks=st["cb"], scales=st["s"]), st["x"], st["go"])
        ref = np.concatenate([gcb.ravel(), gs]).reshape(1, -1)
        return round_to(ref, dtype) if rounded else ref
    if op == "transposed":
        ref = exact_transposed(lin(st["codes"], st["cb"], st["s"]), st["x"])
    elif op == "grouped":
        ends = np.cumsum((0,) + tuple(fout))
        ref = np.concatenate([exact_forward(lin(st["codes"][a:z], st["cb"][i], st["s"][a:z], st["b"][a:z]), x=st["x"])
                              for i, (a, z) in enumerate(zip(ends[:-1], ends[1:]))], axis=1)
    elif op == "routed":
        off = st["off"]
        ref = np.zeros((batch, fout))
        for e in range(ROUTED_E):
            if off[e + 1] > off[e]:
                ref[off[e]:off[e + 1]] = exact_forward(lin(st["codes"][e], st["cb"][e, 0], st["s"][e]),
                                                       x=st["x"][off[e]:off[e + 1]])
    else:
        ref = exact_forward(lin(st["codes"], st["cb"], st["s"], st["b"]), x=st["x"])
    return round_to(ref, dtype)


def _step_models(entry, rounded=True):
    """The model before the first step, then after each of the S rewrites."""
    st, seq = _state(entry)
    st = dict(st)
    out = [_model(entry, st, rounded)]
    for r in seq:
        key, _, host = REWRITES[r]
        st[key] = host(st[key], st)
        out.append(_model(entry, st, rounded))
    return out


def _check_bounds(entry):
    """The lattice stays exact one exponent below its range, where `s.half` takes the scales."""
    name, op, K, nbits, fin, fout, batch, dtype, _, _ = entry
    if op == "wgrad":
        return  # exact_weight_grad asserts its own premise on every step's data
    st, _ = _state(entry)
    e_lo, e_hi = st["e"]
    out = sum(fout) if op == "grouped" else fout
    lattice_bounds(fin, out, K, dtype, e_lo, e_hi + 1, X_MAX, bias=op in ("gemv", "gemm", "grouped"))


@pytest.mark.parametrize("entry", ENTRIES, ids=ENTRY_IDS)
def test_rewrites_have_teeth(entry):
    """Every rewrite changes the exact output in at least TEETH elements: a call that read the operand as it was
    before the kernel just ahead of it cannot match."""
    _check_bounds(entry)
    models = _step_models(entry, rounded=False)
    for i in range(1, len(models)):
        changed = int(np.count_nonzero(models[i] != models[i - 1]))
        assert changed >= TEETH, f"{entry[0]} step {i - 1} ({_state(entry)[1][i - 1]}): only {changed} outputs change"


def _to_dev(st, entry, device):
    dtype = entry[7]
    t = {}
    for k, v in st.items():
        if k in ("e", "raw") or v is None:
            continue
        if k in ("codes", "off", "doff"):
            t[k] = torch.from_numpy(np.ascontiguousarray(v)).to(device)
        else:
            t[k] = torch.from_numpy(np.ascontiguousarray(v, dtype=np.float32)).to(dtype).to(device)
    t.setdefault("b", None)
    return t


def _launch(entry, t, direct_wgrad):
    """One call of the entry point; returns its output tensor(s).  `direct_wgrad`: the weight gradient through the
    C-ABI into zeroed fp32 buffers allocated here, so no zero-fill kernel sits between the rewrite and the call."""
    from aqlm_b200 import _cabi
    from aqlm_b200.inference_kernels import cuda_kernel as ck

    name, op, K, nbits, fin, fout, batch, dtype, _, _ = entry
    if op == "gemv":
        return ck.matmat(t["x"], t["codes"], t["cb"], t["s"], t["b"])
    if op == "gemm":
        return ck.matmat_dequant(t["x"], t["codes"], t["cb"], t["s"], t["b"])
    if op == "grouped":
        return ck.matmat_dequant_grouped(t["x"], t["codes"], t["cb"], t["s"], t["b"], list(fout))
    if op == "routed":
        return ck.matmat_dequant_routed(t["x"], t["codes"], t["cb"], t["s"], t["off"])
    if op == "transposed":
        return ck.matmat_dequant_transposed(t["x"], t["codes"], t["cb"], t["s"])
    if not direct_wgrad:
        gcb, gs = ck.matmat_weight_grad(t["x"], t["go"], t["codes"], t["cb"], t["s"])
        return (gcb, gs)
    gcb, gs = t["wg_slots"].pop(0)
    w = ck.make_weight(t["codes"], t["cb"], t["s"].reshape(-1), None)
    _cabi.check(_cabi.lib().aqlm_b200_matmat_weight_grad(
        ctypes.byref(w), t["x"].data_ptr(), t["go"].data_ptr(), batch, gcb.data_ptr(), gs.data_ptr(),
        t["ws"].data_ptr(), t["ws"].numel(), torch.cuda.current_stream(t["x"].device).cuda_stream))
    return (gcb, gs)


def _as_np(y):
    if isinstance(y, tuple):
        return np.concatenate([v.float().cpu().numpy().ravel() for v in y]).reshape(1, -1)
    return y.float().cpu().numpy().reshape(-1, y.shape[-1])


def run_scenario_a(entry, device=DEV, direct_wgrad=True):
    """The first call (on the initial operands), then S steps of (rewrite kernel, call); ONE synchronize at the end.
    Returns the outputs of every call, as numpy, and the launches the S calls made."""
    from aqlm_b200 import _cabi
    from aqlm_b200.inference_kernels import cuda_kernel as ck

    name, op, K, nbits, fin, fout, batch, dtype, _, _ = entry
    st, seq = _state(entry)
    t = _to_dev(st, entry, device)
    if op == "wgrad" and direct_wgrad:
        w = ck.make_weight(t["codes"], t["cb"], t["s"].reshape(-1), None)
        need = _cabi.lib().aqlm_b200_matmat_weight_grad_workspace_bytes(ctypes.byref(w), batch)
        t["ws"] = torch.zeros(need, dtype=torch.uint8, device=device)
        t["wg_slots"] = [(torch.zeros(st["cb"].shape, dtype=torch.float32, device=device),
                          torch.full((fout,), float("nan"), dtype=torch.float32, device=device)) for _ in range(S + 1)]
    outs = [_launch(entry, t, direct_wgrad)]  # also sizes the workspace, so no step allocates one
    before = _cabi.launch_count()
    for r in seq:
        REWRITES[r][1](t)
        outs.append(_launch(entry, t, direct_wgrad))
    launches = _cabi.launch_count() - before
    torch.cuda.synchronize(device)
    return [_as_np(y) for y in outs], launches, t


@gpu
@pytest.mark.parametrize("pdl", [1, 0], ids=["pdl1", "pdl0"])
@pytest.mark.parametrize("entry", ENTRIES, ids=ENTRY_IDS)
def test_operands_rewritten_by_the_kernel_just_before(entry, pdl):
    name, *_, switches, per_call = entry
    with tunables(pdl=pdl, **switches):
        outs, launches, _ = run_scenario_a(entry)
    assert launches == S * per_call, f"{name}: {launches} launches for {S} calls; the entry took another path"
    for i, (y, ref) in enumerate(zip(outs, _step_models(entry, rounded=False))):
        what = f"{name} PDL={pdl} " + ("first call" if i == 0 else f"step {i - 1} after {_state(entry)[1][i - 1]}")
        assert_exact(y, ref, what)


# ==== B: training steps without a host sync ==========================================================================
T_STEPS = 6
TOL_OUT, TOL_PARAM = 2e-3, 5e-3
MIN_STEP_CHANGE = 0.05  # > 10 * TOL_OUT: a forward that read the previous step's weights fails by a wide margin
# kind -> (K, nbits, in, outs, rows, dtype, lr)
TRAIN = {
    "linear-gemv-4rows": ("linear", 2, 8, 512, (256,), 4, F16, 0.006),
    "linear-gemm-64rows": ("linear", 2, 8, 512, (256,), 64, F16, 0.004),
    "group-2x8": ("group", 2, 8, 256, (128, 64, 64), 64, F16, 0.006),
    "group-1x16": ("group", 1, 16, 256, (128, 64, 64), 64, F16, 0.01),
    "mixtral-2x8": ("mixtral", 2, 8, 64, (64, 64), 24, F16, 1e-4),
}
MIX_E = 4


def _rand_linear(rng, fin, fout, K, nbits, bias):
    """Random quantized linear (float16 values as float32 arrays; codes unsigned)."""
    raw = rng.integers(0, 2 ** nbits, size=(fout, fin // 8, K))
    f16 = lambda a: a.astype(np.float16).astype(np.float32)  # noqa: E731
    return dict(raw=raw, codes=O.pack_int_data(raw.copy(), nbits), cb=f16(rng.standard_normal((K, 2 ** nbits, 1, 8)) / K ** 0.5),
                s=f16(0.75 + 0.5 * rng.random((fout, 1, 1, 1))), b=f16(rng.standard_normal(fout)) if bias else None)


def _train_case(kind):
    """Initial weights, per-step inputs and output gradients of one training scenario (host arrays)."""
    mod, K, nbits, fin, outs, rows, dtype, lr = TRAIN[kind]
    rng = np.random.default_rng(seed_of("train", kind))
    f16 = lambda a: a.astype(np.float16).astype(np.float32)  # noqa: E731
    case = dict(mod=mod, K=K, nbits=nbits, lr=lr, dtype=dtype)
    if mod == "mixtral":
        H, I = outs
        # expert-major, (w1, w2, w3) per expert, as transformers and QuantizedMixtralExperts name them
        case["lins"] = [_rand_linear(rng, *((H, I) if n != "w2" else (I, H)), K, nbits, False)
                        for _ in range(MIX_E) for n in ("w1", "w2", "w3")]
        idx = np.array([0] * 12 + [1] * 8 + [2] * 4)  # skewed; expert 3 gets no token
        case["idx"] = rng.permutation(idx).reshape(rows, 1)
        case["wts"] = f16(rng.choice([0.5, 1.0], size=(rows, 1)))
        out_f = H
    else:
        case["lins"] = [_rand_linear(rng, fin, o, K, nbits, True) for o in outs]
        out_f = sum(outs)
    case["xs"] = [f16(rng.standard_normal((rows, fin))) for _ in range(T_STEPS)]
    case["gos"] = [f16(rng.standard_normal((rows, out_f)) / math.sqrt(rows)) for _ in range(T_STEPS)]
    return case


def _dense_forward(case, params, x):
    """float64 forward of the scenario's module through W = scales * sum_k codebooks[k, codes[:, :, k]]; `params` are
    per linear (codebooks, scales[, bias]) in the module's order.  Returns the output [rows, out] (a group's outputs
    concatenated)."""
    def lin(i, v):
        L = case["lins"][i]
        cb, s = params[i][0], params[i][1]
        raw = torch.from_numpy(L["raw"])
        Wu = sum(cb[k, raw[:, :, k], 0, :] for k in range(case["K"])).reshape(raw.shape[0], -1)
        y = v @ (Wu * s.reshape(-1, 1)).t()
        return y + params[i][2] if len(params[i]) > 2 else y

    if case["mod"] != "mixtral":
        return torch.cat([lin(i, x) for i in range(len(case["lins"]))], dim=1)
    idx = torch.from_numpy(case["idx"][:, 0])
    wts = torch.from_numpy(case["wts"]).double()
    y = torch.zeros((x.shape[0], case["lins"][1]["raw"].shape[0]), dtype=torch.float64)
    for e in range(MIX_E):
        tok = (idx == e).nonzero()[:, 0]
        if tok.numel():
            xe = x[tok]
            y[tok] = lin(3 * e + 1, lin(3 * e, xe) * lin(3 * e + 2, xe)) * wts[tok]
    return y


def replica_train(case):
    """The scenario's T steps on a float64 dense replica: forward, backward of sum(y * go), then SGD; after each update
    the parameters are stored in the module's dtype, as the module stores them.  Returns the outputs per step, the
    final parameters and, per step t >= 1, how far the output moves from the output of the previous step's weights."""
    dt = case["dtype"]
    params = [[torch.from_numpy(L["cb"]).double(), torch.from_numpy(L["s"]).double()] +
              ([torch.from_numpy(L["b"]).double()] if L["b"] is not None else []) for L in case["lins"]]
    outs, moves, prev = [], [], None
    for t in range(T_STEPS):
        x = torch.from_numpy(case["xs"][t]).double()
        req = [[p.clone().requires_grad_() for p in ps] for ps in params]
        y = _dense_forward(case, req, x)
        outs.append(y.detach())
        if prev is not None:
            with torch.no_grad():
                old = _dense_forward(case, prev, x)
            moves.append(((y.detach() - old).norm() / y.detach().norm()).item())
        flat = [p for ps in req for p in ps]
        grads = torch.autograd.grad((y * torch.from_numpy(case["gos"][t]).double()).sum(), flat, allow_unused=True)
        prev = params
        it = iter(grads)
        # an expert without tokens gets no gradient here and a zero one in the module: SGD leaves it unchanged
        params = [[p if g is None else (p - case["lr"] * g).to(dt).double() for p, g in zip(ps, it)] for ps in params]
    return outs, params, moves


def test_training_steps_have_teeth():
    """Each step moves every scenario's output by at least MIN_STEP_CHANGE (more than ten times the output tolerance)
    relative to the output the previous step's weights give on the same input, and the run stays finite."""
    for kind in TRAIN:
        outs, params, moves = replica_train(_train_case(kind))
        assert len(moves) == T_STEPS - 1 and min(moves) >= MIN_STEP_CHANGE, (kind, moves)
        assert max(moves) < 1.0, (kind, moves)
        assert all(torch.isfinite(y).all() for y in outs), kind


def _build_module(case):
    import aqlm_b200
    from aqlm_b200.moe import QuantizedMixtralExperts

    dt, K, nbits = case["dtype"], case["K"], case["nbits"]

    def fill(m, L):
        with torch.no_grad():
            m.codes.copy_(torch.from_numpy(L["codes"]))
            m.codebooks.copy_(torch.from_numpy(L["cb"]))
            m.scales.copy_(torch.from_numpy(L["s"]))
            if L["b"] is not None:
                m.bias.copy_(torch.from_numpy(L["b"]))

    if case["mod"] == "mixtral":
        H, I = case["lins"][1]["raw"].shape[0], case["lins"][0]["raw"].shape[0]
        blk = QuantizedMixtralExperts(MIX_E, H, I, lambda v: v, 8, 1, K, nbits, device=DEV, dtype=dt)
        members = [getattr(blk.expert(e), n) for e in range(MIX_E) for n in ("w1", "w2", "w3")]
        for m, L in zip(members, case["lins"]):
            fill(m, L)
        idx = torch.from_numpy(case["idx"]).to(DEV)
        wts = torch.from_numpy(case["wts"]).to(dt).to(DEV)
        return blk, members, lambda x: blk(x, idx, wts)
    members = []
    for L in case["lins"]:
        fout, fin = L["raw"].shape[0], L["raw"].shape[1] * 8
        m = aqlm_b200.QuantizedLinear(fin, fout, 8, 1, K, nbits, bias=True, device=DEV, dtype=dt)
        fill(m, L)
        members.append(m)
    if case["mod"] == "linear":
        return members[0], members, lambda x: members[0](x)
    grp = aqlm_b200.QuantizedLinearGroup(members)
    assert grp.fused
    return grp, list(grp.members), lambda x: torch.cat(grp(x), dim=-1)


def _rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return ((a - b).norm() / b.norm()).item()


@gpu
@pytest.mark.parametrize("kind", list(TRAIN))
def test_training_steps_without_host_sync(kind):
    """T steps of forward, backward and SGD over codebooks, scales and bias; each forward launches right behind the
    optimizer step that rewrote its weights.  Checked per step against the float64 replica."""
    case = _train_case(kind)
    dt = case["dtype"]
    module, members, fwd = _build_module(case)
    params = [p for m in members for p in (m.codebooks, m.scales, m.bias) if p is not None]
    for p in params:
        p.requires_grad_(True)
    opt = torch.optim.SGD(params, lr=case["lr"])
    xs = [torch.from_numpy(v).to(dt).to(DEV) for v in case["xs"]]
    gos = [torch.from_numpy(v).to(dt).to(DEV) for v in case["gos"]]
    slots = torch.full((T_STEPS,) + tuple(gos[0].shape), float("nan"), dtype=dt, device=DEV)
    torch.cuda.synchronize()
    for t in range(T_STEPS):
        y = fwd(xs[t])
        slots[t].copy_(y.detach())
        y.backward(gos[t])
        opt.step()
        opt.zero_grad(set_to_none=True)
    torch.cuda.synchronize()
    ref_outs, ref_params, _ = replica_train(case)
    for t in range(T_STEPS):
        assert _rel(slots[t], ref_outs[t]) < TOL_OUT, (kind, t, _rel(slots[t], ref_outs[t]))
    mine = [[m.codebooks, m.scales] + ([m.bias] if m.bias is not None else []) for m in members]
    for i, (ps, rs) in enumerate(zip(mine, ref_params)):
        for name, p, r in zip(("codebooks", "scales", "bias"), ps, rs):
            assert _rel(p.detach(), r) < TOL_PARAM, (kind, i, name, _rel(p.detach(), r))


# ==== C: concurrent streams ==========================================================================================
CHAIN = [  # one stream's chain: split-K forward, batch-1 LUT GEMV, split transposed, weight gradient
    ("gemm-1x16-bs64-ks3", "gemm", 1, 16, 1152, 456, 64, F16, {}, 1),
    ("lut-ws-8x8-bs1", "gemv", 8, 8, 1024, 200, 1, F16, {}, 1),
    ("transposed-1x16-bs64-ks3", "transposed", 1, 16, 1088, 456, 64, F16, {}, 1),
    ("wgrad-2x8-bs64", "wgrad", 2, 8, 1152, 200, 64, F16, {}, 1),
]
ROUNDS = 3
N_STREAMS = 3


def _round_inputs(entry, key, n):
    """`n` different activations (or output gradients) for one entry: the lattice draw, then further draws."""
    st, _ = _state(entry)
    rng = np.random.default_rng(seed_of("rounds", entry[0], key, n))
    lo = 2 if entry[1] == "wgrad" else X_MAX
    return [st[key]] + [rng.integers(-lo, lo + 1, size=st[key].shape).astype(np.float32) for _ in range(n - 1)]


def _round_models(entry, key, inputs, rounded):
    st, _ = _state(entry)
    return [_model(entry, dict(st, **{key: v}), rounded) for v in inputs]


def _chain_inputs(stream_i):
    """Per chain entry: the activation inputs of each round (the weight gradient: x and grad_output) for stream i."""
    out = []
    for entry in CHAIN:
        xs = _round_inputs(entry, "x", ROUNDS + stream_i)[stream_i:]
        gos = _round_inputs(entry, "go", ROUNDS + stream_i)[stream_i:] if entry[1] == "wgrad" else None
        out.append((xs, gos))
    return out


def _chain_models(stream_i):
    res = []
    for entry, (xs, gos) in zip(CHAIN, _chain_inputs(stream_i)):
        st, _ = _state(entry)
        res.append([_model(entry, dict(st, x=x, **({"go": g} if gos else {})), True)
                    for x, g in zip(xs, gos or [None] * len(xs))])
    return res


def test_concurrent_and_graph_inputs_have_teeth():
    for i in range(N_STREAMS):
        for entry, models in zip(CHAIN, _chain_models(i)):
            for a, b in zip(models, models[1:]):
                assert int(np.count_nonzero(a != b)) >= TEETH, entry[0]
    for entry in GRAPH_OPS:
        for key in ("g", "e"):
            models = _round_models(entry, "x", _graph_inputs(entry, key), True)
            for a, b in zip(models, models[1:]):
                assert int(np.count_nonzero(a != b)) >= TEETH, (entry[0], key)


def _eager_ws(stream, device=DEV):
    from aqlm_b200.inference_kernels import cuda_kernel as ck

    dev = torch.device(device)
    return ck._WORKSPACES.get((dev.index, stream.cuda_stream))


@gpu
def test_concurrent_streams():
    """Three streams, each with its own chain and data; the host loop interleaves their launches.  The only events
    order each stream behind the upload of its inputs."""
    streams = [torch.cuda.Stream() for _ in range(N_STREAMS)]
    data = []
    for i in range(N_STREAMS):
        per = []
        for entry, (xs, gos) in zip(CHAIN, _chain_inputs(i)):
            t = _to_dev(_state(entry)[0], entry, DEV)
            t["xs"] = [torch.from_numpy(v).to(entry[7]).to(DEV) for v in xs]
            t["gos"] = [torch.from_numpy(v).to(entry[7]).to(DEV) for v in gos] if gos else None
            per.append(t)
        data.append(per)
    uploaded = torch.cuda.Event()
    uploaded.record()
    outs = [[[None] * ROUNDS for _ in CHAIN] for _ in range(N_STREAMS)]
    with tunables(gemm_ksplit=3):
        for s in streams:
            s.wait_event(uploaded)
        for r in range(ROUNDS):
            for j, entry in enumerate(CHAIN):
                for i, s in enumerate(streams):
                    with torch.cuda.stream(s):
                        t = dict(data[i][j], x=data[i][j]["xs"][r])
                        if entry[1] == "wgrad":
                            t["go"] = data[i][j]["gos"][r]
                        outs[i][j][r] = _launch(entry, t, direct_wgrad=False)
        torch.cuda.synchronize()
    for i in range(N_STREAMS):
        for j, (entry, models) in enumerate(zip(CHAIN, _chain_models(i))):
            for r in range(ROUNDS):
                assert_exact(_as_np(outs[i][j][r]), models[r], f"stream {i} {entry[0]} round {r}")
    wss = [_eager_ws(s) for s in streams]
    assert all(ws is not None for ws in wss) and len({ws.data_ptr() for ws in wss}) == N_STREAMS
    for i, ws in enumerate(wss):
        assert int(torch.count_nonzero(ws[:WS_TICKETS])) == 0, f"stream {i}: ticket words left nonzero"


# ==== D: graph replay beside eager work ==============================================================================
GRAPH_OPS = [("lut-ws-8x8-bs1", "gemv", 8, 8, 1024, 200, 1, F16, {}, 1),
             ("gemm-1x16-bs64-ks3", "gemm", 1, 16, 1152, 456, 64, F16, {}, 1)]
REPLAYS = 4


def _graph_inputs(entry, key):
    """Activations of the replays ("g") and of the eager calls ("e"): different draws, same weights."""
    xs = _round_inputs(entry, "x", 2 * REPLAYS)
    return xs[:REPLAYS] if key == "g" else xs[REPLAYS:]


@gpu
def test_graph_replay_beside_eager_work():
    """A graph of the LUT GEMV and a split-K forward replays on a side stream while the default stream runs the same
    ops eagerly on other inputs.  The graph has its own workspace (`_workspace`), so nothing needs to order the replays
    against the eager calls, and nothing does."""
    from aqlm_b200.inference_kernels import cuda_kernel as ck

    side = torch.cuda.Stream()
    with tunables(gemm_ksplit=3):
        ts = [_to_dev(_state(e)[0], e, DEV) for e in GRAPH_OPS]
        gx = [[torch.from_numpy(v).to(e[7]).to(DEV) for v in _graph_inputs(e, "g")] for e in GRAPH_OPS]
        ex = [[torch.from_numpy(v).to(e[7]).to(DEV) for v in _graph_inputs(e, "e")] for e in GRAPH_OPS]
        static = [dict(t, x=t["x"].clone()) for t in ts]
        warm = torch.cuda.Stream()
        warm.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(warm):  # eager warm-up sizes the graph workspace before the capture
            for e, t in zip(GRAPH_OPS, static):
                _launch(e, t, False)
        torch.cuda.current_stream().wait_stream(warm)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            gout = [_launch(e, t, False) for e, t in zip(GRAPH_OPS, static)]
        slots = [torch.full((REPLAYS,) + tuple(y.shape), float("nan"), dtype=y.dtype, device=DEV) for y in gout]
        ready = torch.cuda.Event()
        ready.record()
        side.wait_event(ready)
        eager = [[None] * REPLAYS for _ in GRAPH_OPS]
        for r in range(REPLAYS):
            with torch.cuda.stream(side):
                for j, t in enumerate(static):
                    t["x"].copy_(gx[j][r])
                graph.replay()
                for j, y in enumerate(gout):
                    slots[j][r].copy_(y)
            for j, e in enumerate(GRAPH_OPS):
                eager[j][r] = _launch(e, dict(ts[j], x=ex[j][r]), False)
        torch.cuda.synchronize()
    for j, e in enumerate(GRAPH_OPS):
        gm = _round_models(e, "x", _graph_inputs(e, "g"), True)
        em = _round_models(e, "x", _graph_inputs(e, "e"), True)
        for r in range(REPLAYS):
            assert_exact(_as_np(slots[j][r]), gm[r], f"{e[0]} replay {r}")
            assert_exact(_as_np(eager[j][r]), em[r], f"{e[0]} eager {r}")
    for what, ws in (("eager", _eager_ws(torch.cuda.current_stream())), ("graph", ck._GRAPH_WS[0])):
        assert int(torch.count_nonzero(ws[:WS_TICKETS])) == 0, f"{what} workspace: ticket words left nonzero"


# ==== E: host threads ================================================================================================
# One kernel instantiation, gemv_1x16_kernel<half, 8> (batches 5..8), at a different dynamic shared-memory size per
# thread: the activation tile is 8 x in x 2 bytes.  The batch alone cannot do this on the wgmma GEMM: its N tile is a
# template parameter and its stage count follows from N.  The GEMV has no plan or workspace query that reports its
# shared memory (capi.cu computes it at launch), so `gemv_1x16_smem` restates that formula; the launch count and the
# exact outputs confirm the 1x16 kernel ran.  The shared-memory marks are per process: when an earlier test already
# raised this kernel's attribute above these sizes, no thread sets it, and the test checks concurrent launches only.
# The ensure_smem fix rests on reading the code: no test can force the interleaving that lowered the attribute.
THREAD_IN = [3072, 3328, 3584, 4096]
THREAD_BATCH = [5, 6, 7, 8]
THREAD_OUT, THREAD_CALLS = 256, 10
K_SLICE_CHUNKS = 32  # gemv.cuh kSliceChunks


def gemv_1x16_smem(fin, fout, sm_count, bt=8):
    """A restatement of capi.cu's vec_smem_bytes for the 1x16 GEMV: x tile + per-(row, slice) partials of one CTA."""
    slices = math.ceil(fin // 64 / K_SLICE_CHUNKS)
    return bt * fin * 2 + math.ceil(fout / sm_count) * slices * bt * 4


def _thread_case(i, n):
    entry = (f"thread-{i}", "gemv", 1, 16, THREAD_IN[i], THREAD_OUT, THREAD_BATCH[i], F16, {}, 1)
    return entry, _round_inputs(entry, "x", n)


def test_thread_sizes_differ_and_have_teeth():
    sizes = [gemv_1x16_smem(fin, THREAD_OUT, 132) for fin in THREAD_IN]
    assert len(set(sizes)) == len(sizes) and min(sizes) > 48 * 1024 and max(sizes) <= 227 * 1024
    for i in range(len(THREAD_IN)):
        entry, xs = _thread_case(i, THREAD_CALLS)
        models = _round_models(entry, "x", xs, True)
        for a, b in zip(models, models[1:]):
            assert int(np.count_nonzero(a != b)) >= TEETH


@gpu
def test_host_threads_with_their_own_streams():
    """4 host threads, each with its own stream, make 10 calls each of one GEMV instantiation, each thread at its own
    shared-memory size.  Every call must succeed and every output be exact; the threads are joined before anything is
    asserted."""
    from aqlm_b200 import _cabi

    sm = torch.cuda.get_device_properties(0).multi_processor_count
    sizes = [gemv_1x16_smem(fin, THREAD_OUT, sm) for fin in THREAD_IN]
    assert len(set(sizes)) == len(sizes) and min(sizes) > 48 * 1024
    cases = [_thread_case(i, THREAD_CALLS) for i in range(len(THREAD_IN))]
    tensors = []
    for entry, xs in cases:
        t = _to_dev(_state(entry)[0], entry, DEV)
        t["xs"] = [torch.from_numpy(v).to(F16).to(DEV) for v in xs]
        tensors.append(t)
    torch.cuda.synchronize()
    results = [[None] * THREAD_CALLS for _ in cases]
    errors = []
    barrier = threading.Barrier(len(cases))

    def work(i):
        try:
            s = torch.cuda.Stream()
            barrier.wait()
            with torch.cuda.stream(s):
                for k in range(THREAD_CALLS):
                    results[i][k] = _launch(cases[i][0], dict(tensors[i], x=tensors[i]["xs"][k]), False)
        except BaseException as exc:  # noqa: BLE001 -- reported after the join
            errors.append((i, repr(exc)))
            barrier.abort()

    before = _cabi.launch_count()
    threads = [threading.Thread(target=work, args=(i,)) for i in range(len(cases))]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    torch.cuda.synchronize()
    assert not errors, errors
    assert _cabi.launch_count() - before == len(cases) * THREAD_CALLS
    for i, (entry, xs) in enumerate(cases):
        for k, ref in enumerate(_round_models(entry, "x", xs, True)):
            assert_exact(_as_np(results[i][k]), ref, f"thread {i} call {k}")


# ==== F: a second device =============================================================================================
@gpu
@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_second_device_while_the_first_is_current():
    """Every entry point of A on cuda:1 while cuda:0 is current.  The first call is the largest GEMV of E on cuda:0, then
    the same call on cuda:1: cudaFuncSetAttribute applies to the current device only, so a shared-memory mark shared
    across devices would skip setting the attribute on cuda:1 and that launch would fail."""
    from aqlm_b200.inference_kernels import cuda_kernel as ck

    assert torch.cuda.current_device() == 0
    big, _ = _thread_case(len(THREAD_IN) - 1, 1)
    y0 = _launch(big, _to_dev(_state(big)[0], big, "cuda:0"), False)
    y1 = _launch(big, _to_dev(_state(big)[0], big, "cuda:1"), False)
    torch.cuda.synchronize("cuda:1")
    torch.cuda.synchronize("cuda:0")
    assert y0.device == torch.device("cuda:0") and y1.device == torch.device("cuda:1")
    assert_exact(_as_np(y0), _model(big, _state(big)[0]), "cuda:0 1x16 GEMV")
    assert_exact(_as_np(y1), _model(big, _state(big)[0]), "cuda:1 1x16 GEMV after the same call on cuda:0")
    for entry in ENTRIES:
        with tunables(**entry[8]):
            outs, _, _ = run_scenario_a(entry, device="cuda:1", direct_wgrad=False)
        assert torch.cuda.current_device() == 0
        for i, (y, ref) in enumerate(zip(outs, _step_models(entry))):
            assert_exact(y, ref, f"cuda:1 {entry[0]} call {i}")
    ws = [v for (d, _), v in ck._WORKSPACES.items() if d == 1]
    assert ws and all(v.device == torch.device("cuda:1") for v in ws)
