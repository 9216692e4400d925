"""The backward side at every compiled (n, m) instance x dtype against the float64 oracle: the gradient kernels
(mpcb200_lqr_grad_*), the one-call KKT adjoint (mpcb200_lqr_adjoint_*) on both of its routes, the adjoint's and the
step's input layouts, and the LinDx rollout (mpcb200_rollout_*).

What depends on the instance, and how the tests reach it:
  * the gradient kernels pack 32 // (n+m) problems per warp and four warps per CTA (GradCfg); the outer-product
    kernel decodes a flat store index per warp group and masks the stores of the problems past the batch.  Batch sizes
    come from that layout (grad_layout, layout_batches), and batch element b is pool problem b % K with K coprime to
    the warp and CTA sizes, so every position holds a problem whose oracle answer is known, and neighbouring warps and
    CTAs hold different problems.  Every batch copy of a pool problem must equal that problem solved alone, bit for
    bit;
  * the costate kernel keeps a ring of three tiles (T mod 3) and the outer-product kernel works in chunks of four
    time steps (T mod 4): T in {1, ..., 7, 9} covers every residue of both;
  * F_T = T (a full-length F): dF's last slice must come back exactly 0;
  * the adjoint runs the fused column-pair kernel (2 launches) at pair shapes and the masked step + costate + outer
    product kernels (4 launches) elsewhere, under MPCB200_KERNEL=1, and wherever a pointer is not 16-byte aligned;
  * the instance step kernels copy their tiles in bulk only when every pointer and time stride is 16-byte aligned,
    the large-shape kernels decide per tensor (LB_C ... LB_BOX); a contiguous view at an odd storage offset reaches
    them unchanged and must give the aligned call's outputs bit for bit;
  * the rollout gives a problem n lanes (32 // n per warp, idle lanes at n = 3, 5, 6, 7, 12).
Every output buffer of a C ABI call starts as NaN, so an element a kernel does not write fails the comparison.

Tolerances are the harness's: float64 1e-9 x scale (the rollout 1e-12 x scale); float32 4x the float32 oracle's own
error plus 1e-6 x scale; the bitwise claims are bitwise.  test_zz_coverage_table fails when an instance x dtype
missed any of these paths."""
import pytest
import torch

from oracle import lqr_oracle as orc
from tests.gpu_harness import (DEV, DT, F32, F64, INSTANCES, PAIR_SHAPES, abi_adjoint, abi_grad, abi_rollout,
                               adjoint_case, autograd_backward, batch_rows, check_adjoint, check_routes_agree,
                               check_step_fixed, grad_layout, kernel_env, layout_batches,
                               linear_step_case, misaligned, pool_size, round_through, rollout_layout, staged,
                               step_layout, to_dev, within)
from tests.helpers import gen_problem, maxdiff

pytestmark = pytest.mark.gpu
COVERAGE = {}                       # (n, m, dtype) -> {what: set of values seen}
PARAMS = [(n, m, d) for (n, m) in INSTANCES for d in (F64, F32)]
PIDS = [f"n{n}m{m}_{DT[d]}" for n, m, d in PARAMS]
PAIR_PARAMS = [p for p in PARAMS if p[:2] in PAIR_SHAPES]
PAIR_PIDS = [f"n{n}m{m}_{DT[d]}" for n, m, d in PAIR_PARAMS]
GRAD_T = 5
HORIZONS = (1, 2, 3, 4, 5, 6, 7, 9)              # every residue of T mod 3 and of T mod 4
ADJ_T = 5                                        # the fused adjoint runs at every pair shape and dtype
NAMES = ("dx_init", "dC", "dc", "dF", "df")
BITS = {F32: torch.int32, F64: torch.int64}


def _L():
    from mpc.pytorch_b200 import _lib
    return _lib


def _seen(n, m, dtype, what, value):
    COVERAGE.setdefault((n, m, dtype), {}).setdefault(what, set()).add(value)


def _bits(v):
    return v.view(BITS[v.dtype]) if v.is_floating_point() else v


def _same_bits(tag, a, b, names=NAMES):
    """Outputs a and b (lists or dicts over `names`) bit for bit."""
    for i, name in enumerate(names):
        x, y = (a[i], b[i]) if isinstance(a, list) else (a.get(name), b.get(name))
        if x is None and y is None:
            continue
        assert x is not None and y is not None and x.shape == y.shape, f"{tag}: {name} shapes"
        same = _bits(x) == _bits(y)
        assert bool(same.all()), f"{tag}: {name} differs bitwise at {same.logical_not().nonzero()[:4].tolist()}"


def _pool_batch(case, idx):
    """The batch whose element b is pool problem idx[b]: (P, kw, ref64, ref32) of an adjoint_case."""
    P, kw, ref64, ref32 = case
    sel = lambda d: {k: batch_rows(v, idx) for k, v in d.items()}  # noqa: E731
    refs = lambda r: None if r is None else [batch_rows(v, idx) for v in r]  # noqa: E731
    return sel(P), sel(kw), refs(ref64), refs(ref32)


def _dev(P, dtype):
    return {k: to_dev(v, dtype) for k, v in P.items()}


# ------------------------------------------------------------------------------------------------------------------
# the compiled instances are the ones tested
# ------------------------------------------------------------------------------------------------------------------
def test_instance_list_is_complete():
    assert sorted(_L().supported_pairs()) == sorted(INSTANCES)


# ------------------------------------------------------------------------------------------------------------------
# (a) the gradient kernels, fed the oracle's adjoint solution (dx, du)
# ------------------------------------------------------------------------------------------------------------------
def _grad_call(n, m, T, case, dtype, F_T, with_df):
    """abi_grad (outputs poisoned) on the batch `case` whose F has T slices; F_T = T - 1 hands over F[:T-1]."""
    P, _, ref64, _ = case
    D = _dev(P, dtype)
    F = D["F"][:F_T]
    dx, du = to_dev(ref64[5], dtype), to_dev(ref64[6], dtype)
    return abi_grad(n, m, T, D["C"], D["c"], F, D["x"], D["u"], dx, du, D["wx"], with_df, F_T, poison=True)


def _check_grad(tag, got, case, dtype, T, F_T, with_df):
    """float32: the kernel is fed float32-rounded dx, du, so the yardstick is the float32 oracle's own adjoint."""
    _, _, ref64, ref32 = case
    for i, name in enumerate(NAMES):
        w64, w32 = ref64[i], None if ref32 is None else ref32[i]
        if name == "dF":
            w64, w32 = w64[:F_T], None if w32 is None else w32[:F_T]
            if F_T == T:
                assert bool((got[i][T - 1] == 0).all()), f"{tag}: dF[T-1] of a full-length F is not exactly 0"
        if name == "df" and not with_df:
            assert got[i] is None
            continue
        within(tag, name, got[i], w64, w32, dtype)


@pytest.mark.parametrize("n,m,dtype", PARAMS, ids=PIDS)
def test_grad_kernels_at_every_batch_position(n, m, dtype):
    """T = 5, every batch size of the layout, F_T in {T-1, T} with and without df; every batch copy of a pool problem
    equals that problem solved alone, bit for bit."""
    ppw, W = grad_layout(n, m)
    K = pool_size(ppw, W)
    T = GRAD_T
    pool = adjoint_case(1300 + 10 * n + m, K, T, n, m, dtype, "box", True, T)
    alone = [_grad_call(n, m, T, _pool_batch(pool, torch.tensor([k])), dtype, T, True)[0] for k in range(K)]
    for B in layout_batches(ppw, W, K):
        idx = torch.arange(B) % K
        case = _pool_batch(pool, idx)
        for F_T, with_df in ((T, True), (T - 1, True), (T, False), (T - 1, False)):
            tag = f"grad n{n}m{m} {DT[dtype]} T={T} B={B} F_T={F_T} df={with_df}"
            got, launches = _grad_call(n, m, T, case, dtype, F_T, with_df)
            assert launches == 2, f"{tag}: {launches} launches"
            _check_grad(tag, got, case, dtype, T, F_T, with_df)
            if (F_T, with_df) == (T, True):
                for i, name in enumerate(NAMES):
                    bdim = 0 if i == 0 else 1
                    ref = torch.cat([alone[k][i] for k in idx.tolist()], bdim)
                    _same_bits(f"{tag} vs alone", [got[i]], [ref], (name,))
                _seen(n, m, dtype, "grad_F_T=T", True)
        _seen(n, m, dtype, "grad_B", B)


@pytest.mark.parametrize("n,m,dtype", PARAMS, ids=PIDS)
def test_grad_kernels_at_every_horizon_residue(n, m, dtype):
    """B = W + 1 (a full CTA and one problem), T in {1, ..., 7, 9}, F_T in {T-1, T} with and without df."""
    ppw, W = grad_layout(n, m)
    K = pool_size(ppw, W)
    B = W + 1
    idx = torch.arange(B) % K
    for T in HORIZONS:
        case = _pool_batch(adjoint_case(1400 + 10 * n + m + T, K, T, n, m, dtype, "box", True, T), idx)
        for F_T, with_df in ((T, True), (T - 1, False), (T, False), (T - 1, True)):
            tag = f"grad n{n}m{m} {DT[dtype]} T={T} B={B} F_T={F_T} df={with_df}"
            got, launches = _grad_call(n, m, T, case, dtype, F_T, with_df)
            assert launches == 2, f"{tag}: {launches} launches"
            _check_grad(tag, got, case, dtype, T, F_T, with_df)
        _seen(n, m, dtype, "grad_T", T)


# ------------------------------------------------------------------------------------------------------------------
# (b) the one-call adjoint on both routes
# ------------------------------------------------------------------------------------------------------------------
ADJ_BOUNDS = (None, "box", "tensor")


def _active_fraction(case):
    """Fraction of the controls of the case on a bound (the adjoint's active set)."""
    P, kw, _, _ = case
    u = P["u"]
    lo, hi = (torch.as_tensor(kw[k], dtype=F64).expand_as(u) for k in ("u_lower", "u_upper"))
    return float((((u - lo).abs() <= 1e-8) | ((u - hi).abs() <= 1e-8)).double().mean())


def _routes(n, m):
    """(MPCB200_KERNEL, (ppw, W) of the route's layout) of the adjoint routes: the default and the generic kernel
    forced."""
    grad = (1, grad_layout(n, m))
    if (n, m) in PAIR_SHAPES:
        return [(None, step_layout("pair", n, m, F64)), grad]
    return [(None, grad_layout(n, m)), grad]


def adjoint_launches(n, m, B, dtype, impl):
    """Launches of an adjoint call on fresh tensors: the fused kernel (2) at a pair shape under the default dispatch
    when every time stride of the nested step is a 16-byte multiple (api.cu: bulk_ok), else the 3-launch route (4)."""
    p = n + m
    spans = all(B * k * dtype.itemsize % 16 == 0 for k in (p * p, p, n * p, n, m))
    return 2 if (n, m) in PAIR_SHAPES and impl is None and spans else 4


@pytest.mark.parametrize("n,m,dtype", PARAMS, ids=PIDS)
def test_adjoint_routes_at_every_batch_position(n, m, dtype):
    """Bounds none, scalar and tensor (a strictly partial active set) at every batch size of both routes' layouts:
    each route against the oracle, with its launch count, and the routes against each other; then F_T = T on both."""
    routes = _routes(n, m)
    K = pool_size(*[s for _, lay in routes for s in lay])
    T = ADJ_T
    batches = sorted({B for _, (ppw, W) in routes for B in layout_batches(ppw, W, K)})
    for k, bounds in enumerate(ADJ_BOUNDS):
        with_f = bounds is not None                       # unbounded: has_f = 0, the NaN df buffer stays untouched
        pool = adjoint_case(1500 + 10 * n + m + k, K, T, n, m, dtype, bounds, with_f)
        if bounds is not None:
            frac = _active_fraction(pool)
            assert 0 < frac < 1, f"n{n}m{m} {DT[dtype]} {bounds}: active fraction {frac}"
        for B in batches:
            case = _pool_batch(pool, torch.arange(B) % K)
            got = []
            for impl, _ in routes:
                launches = adjoint_launches(n, m, B, dtype, impl)
                tag = f"adjoint n{n}m{m} {DT[dtype]} T={T} B={B} bounds={bounds} MPCB200_KERNEL={impl}"
                g, nl = run_abi_adjoint_batch(n, m, T, case, dtype, impl)
                assert nl == launches, f"{tag}: {nl} launches"
                check_adjoint(tag, g, case, dtype)
                _seen(n, m, dtype, f"adjoint_{impl}", nl)
                got.append(g)
            check_routes_agree(f"adjoint n{n}m{m} {DT[dtype]} B={B} bounds={bounds} routes", got[0], got[1], case,
                               dtype)
    B = 4 * (grad_layout(n, m)[1] // 4 + 1)                # past a CTA, and the fused route where it applies
    pool = adjoint_case(1600 + 10 * n + m, K, T, n, m, dtype, "tensor", True, T)
    case = _pool_batch(pool, torch.arange(B) % K)
    got = []
    for impl, _ in routes:
        launches = adjoint_launches(n, m, B, dtype, impl)
        tag = f"adjoint n{n}m{m} {DT[dtype]} T={T} B={B} F_T=T MPCB200_KERNEL={impl}"
        g, nl = run_abi_adjoint_batch(n, m, T, case, dtype, impl, F_T=T)
        assert nl == launches, f"{tag}: {nl} launches"
        assert bool((g[3][T - 1] == 0).all()), f"{tag}: dF[T-1] of a full-length F is not exactly 0"
        check_adjoint(tag, g, case, dtype)
        _seen(n, m, dtype, "adjoint_F_T=T", nl)
        got.append(g)
    check_routes_agree(f"adjoint n{n}m{m} {DT[dtype]} F_T=T routes", got[0], got[1], case, dtype)


def run_abi_adjoint_batch(n, m, T, case, dtype, impl, F_T=None):
    """abi_adjoint (outputs poisoned) on a pool batch; F_T None: F[:T-1] of an F that may carry T slices."""
    P, kw = case[:2]
    D = _dev(P, dtype)
    F_T = T - 1 if F_T is None else F_T
    with kernel_env(impl):
        return abi_adjoint(n, m, T, D["C"], D["c"], D["F"][:F_T], D["x"], D["u"], D["wx"], D["wu"],
                           to_dev(kw.get("u_lower"), dtype), to_dev(kw.get("u_upper"), dtype), P["f"] is not None,
                           F_T, poison=True)


# one shape per dtype: the 3-launch route at a shape no other backward test reaches, and the fused route
BACKWARD_ONE_CALL = [(3, 2, F64), (6, 2, F32)]


@pytest.mark.parametrize("n,m,dtype", BACKWARD_ONE_CALL, ids=[f"n{n}m{m}_{DT[d]}" for n, m, d in BACKWARD_ONE_CALL])
def test_lqrstep_backward_is_the_adjoint_call(n, m, dtype):
    """LQRStepFn.backward is the one mpcb200_lqr_adjoint_* call: the same launches and the same gradients, bit for
    bit, as the C ABI call on the same input, and both against the oracle."""
    ppw, W = grad_layout(n, m)
    K, B = pool_size(ppw, W), 4 * (W // 4 + 1)
    launches = adjoint_launches(n, m, B, dtype, None)
    case = _pool_batch(adjoint_case(1700 + 10 * n + m, K, ADJ_T, n, m, dtype, "tensor", True), torch.arange(B) % K)
    tag = f"LQRStepFn.backward n{n}m{m} {DT[dtype]} B={B}"
    auto, l_auto = autograd_backward(n, m, ADJ_T, *case[:2], dtype)
    assert l_auto == launches, f"{tag}: {l_auto} launches"
    check_adjoint(tag, auto, case, dtype)
    abi, l_abi = run_abi_adjoint_batch(n, m, ADJ_T, case, dtype, None)
    assert l_abi == launches, f"{tag}: C ABI {l_abi} launches"
    _same_bits(tag + " vs C ABI", auto, abi)


# ------------------------------------------------------------------------------------------------------------------
# (c) the adjoint's input layouts
# ------------------------------------------------------------------------------------------------------------------
def _layout_B(n, m):
    """A multiple of 4 (every time stride a 16-byte multiple, so the aligned call takes the fused route): two warps
    of the fused kernel and a tail where it packs fewer than 8 problems per warp, else 12 (one partial warp)."""
    ppw = step_layout("pair", n, m, F64)[0]
    return ((2 * ppw + 2 + 3) // 4) * 4 if ppw < 8 else 12


@pytest.mark.parametrize("n,m,dtype", PAIR_PARAMS, ids=PAIR_PIDS)
def test_adjoint_input_layouts(n, m, dtype):
    """One tensor at a time: stride-0 C, stride-0 F, c with a 2x time stride and a misaligned dl_dx or dl_du keep the
    fused route and its outputs bit for bit; a misaligned C, c or new_u sends the call to the 3-launch route, which
    agrees with the fused one."""
    T, B = ADJ_T, _layout_B(n, m)
    K = pool_size(step_layout("pair", n, m, F64)[0])
    case = _pool_batch(adjoint_case(1800 + 10 * n + m, K, T, n, m, dtype, "tensor", True), torch.arange(B) % K)
    P, kw = case[:2]
    D = _dev(P, dtype)
    lo, hi = to_dev(kw["u_lower"], dtype), to_dev(kw["u_upper"], dtype)

    def call(**over):
        A = dict(D, **over)
        return abi_adjoint(n, m, T, A["C"], A["c"], A["F"], A["x"], A["u"], A["wx"], A["wu"], lo, hi, True,
                           poison=True)

    base, nl = call()
    tag = f"adjoint layouts n{n}m{m} {DT[dtype]} T={T} B={B}"
    assert nl == 2, f"{tag}: {nl} launches"
    check_adjoint(tag, base, case, dtype)
    C0 = D["C"][:1].expand(T, *D["C"].shape[1:])
    F0 = D["F"][:1].expand(T - 1, *D["F"].shape[1:])
    c2 = torch.zeros(2 * T, *D["c"].shape[1:], dtype=D["c"].dtype, device=DEV)
    c2[::2] = D["c"]
    p = n + m
    assert staged(C0, dtype)[1] == -1 and staged(F0, dtype)[1] == -1 and staged(c2[::2], dtype)[1] == 2 * B * p
    for what, over, dense in (("stride-0 C", dict(C=C0), dict(C=C0.contiguous())),
                              ("stride-0 F", dict(F=F0), dict(F=F0.contiguous())),
                              ("c with a 2x time stride", dict(c=c2[::2]), {}),
                              ("misaligned dl_dx", dict(wx=misaligned(D["wx"])), {}),
                              ("misaligned dl_du", dict(wu=misaligned(D["wu"])), {})):
        got, nl = call(**over)
        assert nl == 2, f"{tag} {what}: {nl} launches"
        want, nl = call(**dense) if dense else (base, 2)
        assert nl == 2
        _same_bits(f"{tag} {what}", got, want)
        _seen(n, m, dtype, "adjoint_layout", what)
    for what, over in (("misaligned C", dict(C=misaligned(D["C"]))), ("misaligned c", dict(c=misaligned(D["c"]))),
                       ("misaligned new_u", dict(u=misaligned(D["u"])))):
        got, nl = call(**over)
        assert nl == 4, f"{tag} {what}: {nl} launches, not the 3-launch route"
        check_adjoint(f"{tag} {what}", got, case, dtype)
        check_routes_agree(f"{tag} {what} vs aligned", got, base, case, dtype)
        _seen(n, m, dtype, "adjoint_layout", what)


# ------------------------------------------------------------------------------------------------------------------
# (d) the step kernels under per-tensor misalignment
# ------------------------------------------------------------------------------------------------------------------
STEP_TENSORS = ("C", "c", "F", "f", "cur_x", "cur_u", "x_init", "u_lower")
_KEY = {"cur_x": "x", "cur_u": "u", "x_init": "x0"}
STEP_OUTPUTS = ("new_x", "new_u", "costs", "alphas", "full_du_norm", "Ks", "ks", "qp_iters", "free_mask", "status")


def _step(n, m, T, D, kw, impl):
    from mpc.pytorch_b200.step import lqr_step_raw
    with kernel_env(impl):
        o = lqr_step_raw(n, m, T, D["x0"], D["C"], D["c"], D["F"], D["f"], D["x"], D["u"], want_gains=True, **kw)
        plan = _L().last_step_plan()
    torch.cuda.synchronize()
    return {k: v.cpu() for k, v in o.items() if v is not None}, plan


def misaligned_step_inputs(D, kw, which):
    """The step inputs D (device tensors) and options kw with the tensor `which` (a name of STEP_TENSORS) replaced
    by a misaligned copy."""
    D, kw = dict(D), dict(kw)
    if which == "u_lower":
        kw["u_lower"] = misaligned(kw["u_lower"])
    else:
        k = _KEY.get(which, which)
        D[k] = misaligned(D[k])
    return D, kw


def step_misalign_B(n, m, dtype):
    """A multiple of 4 past the generic kernel's first CTA: every span and time stride is a 16-byte multiple."""
    W = step_layout("generic", n, m, dtype)[1]
    return 4 * (W // 4 + 1)


@pytest.mark.parametrize("n,m,dtype", PARAMS, ids=PIDS)
def test_step_kernels_under_misalignment(n, m, dtype):
    """The generic kernel (default dispatch at a generic-only shape, MPCB200_KERNEL=1 at a pair shape) with one
    tensor at a time misaligned: every output bit for bit the aligned call's.  At a pair shape the default dispatch
    runs the generic kernel for a misaligned input, bit for bit the aligned MPCB200_KERNEL=1 call, where it runs the
    column-pair kernel for the aligned one."""
    T, B = 4, step_misalign_B(n, m, dtype)
    case = linear_step_case(1900 + 10 * n + m, B, T, n, m, dtype, "boxT")
    P, kw, o64 = case[:3]
    D, kw_d = _dev(P, dtype), {k: to_dev(v, dtype) for k, v in kw.items()}
    pair = (n, m) in PAIR_SHAPES
    impl = 1 if pair else None
    base, plan = _step(n, m, T, D, kw_d, impl)
    L = _L()
    assert plan & L.PLAN_GENERIC, f"n{n}m{m} {DT[dtype]}: plan {plan}"
    if dtype == F64:
        check_step_fixed(f"misalign n{n}m{m} {DT[dtype]} aligned", base, o64, kw, dtype)
    pair_default = pair and bool(_step(n, m, T, D, kw_d, None)[1] & L.PLAN_PAIR)
    for which in STEP_TENSORS:
        Dm, kwm = misaligned_step_inputs(D, kw_d, which)
        tag = f"step n{n}m{m} {DT[dtype]} B={B} misaligned {which}"
        got, p = _step(n, m, T, Dm, kwm, impl)
        assert p == plan, f"{tag}: plan {p}, aligned {plan}"
        _same_bits(tag, got, base, STEP_OUTPUTS)
        if pair_default:
            got, p = _step(n, m, T, Dm, kwm, None)
            assert p & L.PLAN_GENERIC, f"{tag}: the default dispatch ran plan {p}, not the generic kernel"
            _same_bits(tag + " default dispatch", got, base, STEP_OUTPUTS)
        _seen(n, m, dtype, "step_misaligned", which)


# (n, m, dtype) of the large-shape kernels at which every per-problem span is a 16-byte multiple
LARGE_MISALIGN = [(20, 4, F32), (24, 8, F64)]
LARGE_TENSORS = ("C", "c", "F", "f", "cur_x", "cur_u", "u_lower")


@pytest.mark.parametrize("n,m,dtype", LARGE_MISALIGN, ids=[f"n{n}m{m}_{DT[d]}" for n, m, d in LARGE_MISALIGN])
def test_large_step_under_misalignment(n, m, dtype):
    """Each misaligned tensor moves one tensor from the bulk copy to the element copy (one LB_* bit): every output bit
    for bit the aligned call's, which is compared with the float64 oracle."""
    T, B = 4, 5
    case = linear_step_case(2000 + n + m, B, T, n, m, dtype, "boxT")
    P, kw, o64 = case[:3]
    D, kw_d = _dev(P, dtype), {k: to_dev(v, dtype) for k, v in kw.items()}
    base, plan = _step(n, m, T, D, kw_d, None)
    assert plan == _L().PLAN_LARGE, f"n{n}m{m}: plan {plan}, not the large-shape kernels"
    tag = f"large n{n}m{m} {DT[dtype]} aligned"
    if dtype == F64:
        check_step_fixed(tag, base, o64, kw, dtype)
    else:       # float32: a control at its bound may be clamped or not by round-off; the trajectory to 2e-4
        scale = max(1.0, float(o64.new_x.abs().max()))
        for k in ("new_x", "new_u", "Ks", "ks"):
            assert maxdiff(base[k], getattr(o64, k)) <= 2e-4 * scale, f"{tag}: {k}"
        assert maxdiff(base["costs"], o64.costs) <= 3e-4 * max(1.0, float(o64.costs.abs().max())), f"{tag}: costs"
    for which in LARGE_TENSORS:
        Dm, kwm = misaligned_step_inputs(D, kw_d, which)
        got, p = _step(n, m, T, Dm, kwm, None)
        assert p == plan
        _same_bits(f"large n{n}m{m} {DT[dtype]} misaligned {which}", got, base, STEP_OUTPUTS)


# ------------------------------------------------------------------------------------------------------------------
# (e) the LinDx rollout
# ------------------------------------------------------------------------------------------------------------------
ROLLOUT_T = (1, 2, 3, 17)


def _rollout_inputs(seed, B, T, n, m, dtype):
    """x0, u, F [T slices], f [T-1 slices] (float64, rounded through dtype); time-varying F and f."""
    C, c, F, f, x0 = gen_problem(seed, B, T + 1, n, m, F64, time_varying=True)
    u = torch.randn(T, B, m, generator=torch.Generator().manual_seed(seed), dtype=F64)
    return [round_through(t, dtype) for t in (x0, u, 0.9 * F[:T], f[:T - 1])]


@pytest.mark.parametrize("n,m,dtype", PARAMS, ids=PIDS)
def test_rollout_at_every_batch_position(n, m, dtype):
    """Every batch size of the layout, T in {1, 2, 3, 17}: with and without f, F_T in {T-1, T}, a misaligned F and,
    from T = 3 on, a stride-0 F (time-invariant code), against orc.get_traj."""
    ppw, W = rollout_layout(n)
    lo = lambda t: None if t is None else t.float()  # noqa: E731
    for B in layout_batches(ppw, W):
        for T in ROLLOUT_T:
            x0, u, F, f = _rollout_inputs(2100 + 10 * n + m + T, B, T, n, m, dtype)
            Fd = to_dev(F, dtype)
            variants = [("f, F_T=T-1", Fd[:T - 1], f, F[:T - 1]), ("no f, F_T=T", Fd, None, F),
                        ("misaligned F, F_T=T", misaligned(Fd), f, F)]
            if T > 2:
                # two or more slices (one is contiguous, hence dense), expanded on the device: a copy of an expanded
                # tensor to the device or to another dtype would be dense
                F1 = Fd[:1].expand(T - 1, *Fd.shape[1:])
                assert staged(F1, dtype)[1] == -1, "the stride-0 F does not reach the kernel as time invariant"
                variants.append(("stride-0 F", F1, f, F[:1].expand(T - 1, *F.shape[1:])))
            for what, Fk, fk, F_orc in variants:
                tag = f"rollout n{n}m{m} {DT[dtype]} B={B} T={T} {what}"
                got = abi_rollout(n, m, T, Fk, to_dev(fk, dtype), to_dev(x0, dtype), to_dev(u, dtype), poison=True)
                w64 = orc.get_traj(T, u, x0, F_orc, fk)
                w32 = orc.get_traj(T, lo(u), lo(x0), lo(F_orc), lo(fk)) if dtype == F32 else None
                within(tag, "x", got, w64, w32, dtype, tol64=1e-12)
                _seen(n, m, dtype, "rollout", (B, T, what.split(",")[0]))


# ------------------------------------------------------------------------------------------------------------------
# coverage: every instance x dtype reached every path (runs last)
# ------------------------------------------------------------------------------------------------------------------
def test_zz_coverage_table():
    if not COVERAGE:
        pytest.skip("no test of this module ran")
    rows, missing = [], []
    for n, m, dtype in PARAMS:
        cov = COVERAGE.get((n, m, dtype), {})
        pair = (n, m) in PAIR_SHAPES
        ppw, W = grad_layout(n, m)
        Ts = cov.get("grad_T", set())
        residues = {(T % 3, T % 4) for T in Ts}
        need = {
            "grad at every batch size": set(layout_batches(ppw, W, pool_size(ppw, W))) <= cov.get("grad_B", set()),
            "grad at every T mod 3, T mod 4": {r for r, _ in residues} == {0, 1, 2}
            and {r for _, r in residues} == {0, 1, 2, 3},
            "grad F_T=T": bool(cov.get("grad_F_T=T")),
            "adjoint default route": (2 if pair else 4) in cov.get("adjoint_None", set()),
            "adjoint 3-launch route": cov.get("adjoint_1") == {4},
            "adjoint F_T=T on both routes": cov.get("adjoint_F_T=T", set()) == ({2, 4} if pair else {4}),
            "step misaligned tensors": cov.get("step_misaligned", set()) == set(STEP_TENSORS),
            "rollout": len(cov.get("rollout", ())) == len(layout_batches(*rollout_layout(n)))
            * (3 * len(ROLLOUT_T) + sum(T > 2 for T in ROLLOUT_T)),      # stride-0 F from T = 3 on
        }
        if pair:
            need["adjoint layouts"] = len(cov.get("adjoint_layout", ())) == 8
        for k, ok in need.items():
            if not ok:
                missing.append(f"n{n}m{m} {DT[dtype]}: {k}")
        cell = lambda k: "x" if need.get(k) else ("-" if k not in need else "MISSING")  # noqa: E731
        rows.append(f"| ({n},{m}) {DT[dtype]} | {ppw}/{W} | " + " | ".join(cell(k) for k in need_keys()) + " |")
    print("\n| instance | grad PPW/W | " + " | ".join(need_keys()) + " |\n|" + "---|" * (2 + len(need_keys())))
    print("\n".join(rows))
    assert not missing, "\n".join(missing)


def need_keys():
    return ("grad at every batch size", "grad at every T mod 3, T mod 4", "grad F_T=T", "adjoint default route",
            "adjoint 3-launch route", "adjoint F_T=T on both routes", "adjoint layouts", "step misaligned tensors",
            "rollout")
