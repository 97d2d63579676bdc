"""Adaptive Dormand–Prince (the reference's default solver).  torchdiffeq is absent: the oracle restates its
published algorithm and is itself sanity-checked on an ODE with a closed-form solution (CPU); the CUDA driver
is compared against the oracle on the estimator's vector field (GPU).  Parity with torchdiffeq: UNPINNED."""
import math

import pytest
import torch

from conftest import rel_errs
from oracle import adaptive_ref as AD
from oracle import estimator_ref as R
from oracle import cases, weights


def test_oracle_on_closed_form_ode():
    f = lambda t, y: -y + torch.sin(3 * t)
    out, stats = AD.odeint_dopri5(f, torch.ones(3), 1.0, 1e-7, 1e-7)
    exact = math.exp(-1) * 1.3 + (math.sin(3) - 3 * math.cos(3)) / 10
    assert abs(float(out[0]) - exact) < 5e-6
    assert stats["accepted"] >= 3 and stats["nfe"] == 2 + 6 * (stats["accepted"] + stats["rejected"])


def test_tableau_matches_an_independent_implementation():
    """The 5th-order Dormand–Prince tableau (nodes, stage matrix, solution weights) against scipy's RK45, an
    independent implementation of the same published method that IS installed here.  (The embedded 4th-order
    weights differ on purpose: torchdiffeq uses Shampine's variant, last error coefficient -1/60; scipy the
    classic 1/40 — so step sequences are not comparable one to one, only the solutions are.)"""
    import numpy as np
    from scipy.integrate._ivp.rk import RK45
    assert np.allclose(RK45.C[1:], AD.ALPHA[:5]) and AD.ALPHA[5] == 1.0
    for i, row in enumerate(AD.BETA[:5]):
        assert np.allclose(RK45.A[i + 1][:len(row)], row, rtol=0, atol=1e-15)
    assert np.allclose(RK45.B, AD.C_SOL[:6], rtol=0, atol=1e-15) and AD.C_SOL[6] == 0
    assert np.allclose(AD.BETA[5], AD.C_SOL[:6])                      # FSAL: last stage input = the solution
    assert abs(sum(AD.C_ERROR)) < 1e-15                               # both weight sets sum to one


def test_bosh3_tableau_matches_scipy_rk23():
    """Bogacki–Shampine 3(2): nodes, stage matrix, 3rd-order weights AND the embedded error weights against scipy's RK23
    (scipy stores E = low - high, torchdiffeq high - low: equal up to the sign, which the error norm ignores)."""
    import numpy as np
    from scipy.integrate._ivp.rk import RK23
    tb = AD.TABLEAUS["bosh3"]
    assert np.allclose(RK23.C[1:], tb.alpha[:2]) and tb.alpha[2] == 1.0
    for i, row in enumerate(tb.beta[:2]):
        assert np.allclose(RK23.A[i + 1][:len(row)], row, rtol=0, atol=1e-15)
    assert np.allclose(RK23.B, tb.c_sol[:3], rtol=0, atol=1e-15) and tb.c_sol[3] == 0
    assert np.allclose(tb.beta[2], tb.c_sol[:3])                      # FSAL
    assert np.allclose(np.abs(RK23.E), np.abs(tb.c_error), rtol=0, atol=1e-15)
    assert np.allclose(RK23.E, -np.asarray(tb.c_error), rtol=0, atol=1e-15)


def test_oracle_solution_agrees_with_scipy_rk45():
    """Same nonlinear system, same tolerances: both adaptive solvers must land on the same solution to a few times
    the tolerance, with step counts of the same order."""
    import numpy as np
    from scipy.integrate import solve_ivp

    def rhs_np(t, y):
        return np.array([y[1], -np.sin(y[0]) - 0.3 * y[1] + np.cos(2.0 * t), -0.5 * y[2] + y[0] * y[1]])

    def rhs_t(t, y):
        return torch.stack([y[1], -torch.sin(y[0]) - 0.3 * y[1] + torch.cos(2.0 * t), -0.5 * y[2] + y[0] * y[1]])

    y0 = [1.0, 0.0, 0.5]
    sol = solve_ivp(rhs_np, (0.0, 1.0), y0, method="RK45", rtol=1e-6, atol=1e-6)
    out, stats = AD.odeint_dopri5(rhs_t, torch.tensor(y0, dtype=torch.float32), 1.0, 1e-6, 1e-6)
    assert np.abs(out.numpy() - sol.y[:, -1]).max() < 2e-5
    assert 0.5 * len(sol.t) <= stats["accepted"] + 1 <= 2.0 * len(sol.t)


def _order_conditions(tb, weights, p):
    """Residuals of the Runge-Kutta order conditions up to order p (<= 3) for solution weights ``weights`` over the
    S+1 stage derivatives (stage 0 at c = 0, stage i+1 at c = alpha[i] with row beta[i])."""
    n = tb.stages + 1
    c = [0.0] + list(tb.alpha)
    A = [[0.0] * n for _ in range(n)]
    for i, row in enumerate(tb.beta):
        for j, v in enumerate(row):
            A[i + 1][j] = v
    res = [abs(sum(weights) - 1.0)]
    if p >= 2:
        res.append(abs(sum(w * ci for w, ci in zip(weights, c)) - 0.5))
    if p >= 3:
        res.append(abs(sum(w * ci * ci for w, ci in zip(weights, c)) - 1 / 3))
        res.append(abs(sum(weights[i] * A[i][j] * c[j] for i in range(n) for j in range(n)) - 1 / 6))
    return max(res)


@pytest.mark.parametrize("method,p_sol,p_emb", [("bosh3", 3, 2), ("fehlberg2", 2, 1), ("adaptive_heun", 2, 1), ("dopri5", 3, 3)])
def test_embedded_pairs_satisfy_their_order_conditions(method, p_sol, p_emb):
    """The restated tableaux (torchdiffeq bosh3.py / fehlberg2.py / adaptive_heun.py, from the published pairs) are
    consistent Runge-Kutta pairs: the solution weights meet the order conditions of the stated order, the embedded
    weights (c_sol - c_error) those of one order less, every row of beta sums to its node."""
    tb = AD.TABLEAUS[method]
    assert _order_conditions(tb, list(tb.c_sol), p_sol) < 1e-14
    emb = [a - b for a, b in zip(tb.c_sol, tb.c_error)]
    assert _order_conditions(tb, emb, p_emb) < 1e-14
    for al, row in zip(tb.alpha, tb.beta):
        assert abs(sum(row) - al) < 1e-15
    assert abs(sum(tb.c_error)) < 1e-15 and len(tb.c_mid) == tb.stages + 1
    assert tb.sol_is_last_stage == (method in ("dopri5", "bosh3"))


@pytest.mark.parametrize("method,tol", [("bosh3", 2e-5), ("fehlberg2", 2e-4), ("adaptive_heun", 2e-5)])
def test_other_adaptive_tableaux_on_closed_form_ode(method, tol):
    f = lambda t, y: -y + torch.sin(3 * t)
    out, stats = AD.odeint_adaptive(f, torch.ones(3), method, 1.0, 1e-6, 1e-6)
    exact = math.exp(-1) * 1.3 + (math.sin(3) - 3 * math.cos(3)) / 10
    assert abs(float(out[0]) - exact) < tol, (method, float(out[0]) - exact, stats)
    assert stats["nfe"] == 2 + AD.TABLEAUS[method].stages * (stats["accepted"] + stats["rejected"])


def test_method_strings_of_the_reference_ui():
    """webui.py:110 offers dopri5, euler, midpoint, rk4, implicit_adams, bosh3, fehlberg2, adaptive_heun: all but the
    multistep Adams method map to a built solver; that one raises a ValueError naming the alternatives."""
    from stabletts_b200.flow_matching import _method_id, _ADAPTIVE, ST_ADAPTIVE
    from stabletts_b200 import _lib
    for name in ("dopri5", "bosh3", "fehlberg2", "adaptive_heun", None):
        assert _method_id(name) == ST_ADAPTIVE and name in _ADAPTIVE
    assert _ADAPTIVE["bosh3"] == _lib.ST_ADAPT_BOSH3 and _ADAPTIVE["adaptive_heun"] == _lib.ST_ADAPT_HEUN
    for name in ("euler", "midpoint", "rk4"):
        assert _method_id(name) >= 0
    with pytest.raises(ValueError, match="not built"):
        _method_id("implicit_adams")
    with pytest.raises(ValueError):
        _method_id("no_such_solver")


@pytest.mark.gpu
def test_cuda_adaptive_vs_oracle():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import __graft_entry__ as ge
    ge.build()
    from stabletts_b200 import CFMDecoder
    dev = torch.device("cuda:0")
    n_mel = 80
    st = weights.make_state(cases.WEIGHT_SEED, n_mel)
    # damp the (random-weight) vector field so the solve needs tens, not hundreds, of steps
    for k in list(st):
        if k.startswith("final_proj"):
            st[k] = st[k] * 0.05
    m = CFMDecoder(n_mel, n_mel, 256, n_mel, 1024, 4, 6, 3, 0.1, 256).eval()
    m.estimator.load_state_dict(st, strict=True)
    m = m.to(dev)
    inp = weights.make_inputs(61, [48, 31], 48, n_mel)
    fs, fc = weights.make_cfg_params(cases.CFG_SEED, n_mel)
    z = inp["x"]
    g = lambda t, y: R.cfg_estimator(st, t, y, inp["mask"], inp["mu"], inp["c"], fs, fc, 2.0)
    with torch.inference_mode():
        ref, stats = AD.odeint_dopri5(g, z, 1.0)
    kw = dict(fake_speaker=fs.to(dev), fake_content=fc.to(dev), cfg_strength=2.0)
    out = m(inp["mu"].to(dev), inp["mask"].to(dev), 10, 1.0, inp["c"].to(dev), None, kw, z=z.to(dev))
    got = m.last_solver_stats
    e = rel_errs(out, ref)
    # both sides solve the same ODE to rtol = atol = 1e-5; step sequences may differ by a borderline accept
    assert max(e) < 1e-3, (e, stats, got)
    assert abs(got["accepted"] - stats["accepted"]) <= max(2, stats["accepted"] // 10), (stats, got)
    assert got["nfe"] == 2 + 6 * (got["accepted"] + got["rejected"])


@pytest.mark.gpu
@pytest.mark.parametrize("method,stages", [("bosh3", 3), ("fehlberg2", 2), ("adaptive_heun", 1)])
def test_cuda_other_adaptive_solvers_vs_oracle(method, stages):
    """bosh3 / fehlberg2 / adaptive_heun through CFMDecoder.forward(solver=...) against the oracle restatement on the
    estimator's (damped) vector field.  Low-order pairs at rtol = atol = 1e-5 take many steps: a short utterance."""
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import __graft_entry__ as ge
    ge.build()
    from stabletts_b200 import CFMDecoder
    dev = torch.device("cuda:0")
    n_mel = 80
    st = weights.make_state(cases.WEIGHT_SEED, n_mel)
    for k in list(st):
        if k.startswith("final_proj"):
            st[k] = st[k] * 0.02
    m = CFMDecoder(n_mel, n_mel, 256, n_mel, 1024, 4, 6, 3, 0.1, 256).eval()
    m.estimator.load_state_dict(st, strict=True)
    m = m.to(dev)
    inp = weights.make_inputs(62, [24, 17], 24, n_mel)
    z = inp["x"]
    g = lambda t, y: R.estimator_forward(st, t, y, inp["mask"], inp["mu"], inp["c"])
    with torch.inference_mode():
        ref, stats = AD.odeint_adaptive(g, z, method)
    out = m(inp["mu"].to(dev), inp["mask"].to(dev), 10, 1.0, inp["c"].to(dev), method, None, z=z.to(dev))
    got = m.last_solver_stats
    e = rel_errs(out, ref)
    assert max(e) < 1e-3, (method, e, stats, got)
    assert abs(got["accepted"] - stats["accepted"]) <= max(2, stats["accepted"] // 10), (stats, got)
    assert got["nfe"] == 2 + stages * (got["accepted"] + got["rejected"]) and got["solver"] == method


@pytest.mark.gpu
def test_adaptive_solves_ignore_the_two_pass_precision_mode():
    """The adaptive controller compares an error estimate with rtol = atol = 1e-5, below the two-pass FFN mode's evaluation
    noise: st_solve_adaptive_ex therefore evaluates the vector field with three passes whatever the handle's mode.  At a
    batch large enough for the 256-channel GEMM tiles the default-mode result must be BIT-identical to the bf16x3-mode result (and the
    fixed-grid solve of the same problem must differ between the modes: proof that the mode is otherwise active)."""
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import __graft_entry__ as ge
    ge.build()
    from stabletts_b200 import CFMDecoder
    dev = torch.device("cuda:0")
    st = weights.make_state(cases.WEIGHT_SEED, 80)
    for k in list(st):
        if k.startswith("final_proj"):
            st[k] = st[k] * 0.05
    m = CFMDecoder(80, 80, 256, 80, 1024, 4, 6, 3, 0.1, 256).eval()
    m.estimator.load_state_dict(st, strict=True)
    m = m.to(dev)
    inp = weights.make_inputs(63, [1024] * 19 + [700], 1024, 80)
    a = [inp[k].to(dev) for k in ("mu", "mask", "c", "x")]
    outs, fixed = {}, {}
    for mode in ("ffn_fp16x2", "bf16x3"):
        m.estimator.set_precision(mode)
        outs[mode] = m(a[0], a[1], 10, 1.0, a[2], None, None, z=a[3]).cpu()
        stats = dict(m.last_solver_stats)
        fixed[mode] = m(a[0], a[1], 2, 1.0, a[2], "euler", None, z=a[3]).cpu()
    assert torch.equal(outs["ffn_fp16x2"], outs["bf16x3"]), stats
    assert not torch.equal(fixed["ffn_fp16x2"], fixed["bf16x3"])
    assert stats["accepted"] >= 2 and torch.isfinite(outs["bf16x3"]).all()
