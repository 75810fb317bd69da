"""GPU parity: the GCBF+ train step (losses, hand-written backward, clip + AdamW) vs the
oracle's torch-autograd restatement of gcbf_plus.py:354-447 in float64.
Tolerance: gradients within 2e-4 of the float64 reference relative to the gradient's max
magnitude per tensor (fp32 accumulation over edges/agents, atomics order); losses 1e-5."""
import numpy as np
import pytest
import torch

from helpers import (oracle_env, oracle_obstacles, oracle_params, product_algo, product_env, product_obstacles,
                     random_scene)

pytestmark = pytest.mark.gpu

# the last two rows: gradient parity at a size where every agent has real neighbours and several row tiles / CTAs
# contribute to each dW (VERDICT r1): DoubleIntegrator N=64, B=4 and LinearDrone N=32, B=3 on the oracle's sparse graph
CASES = [("DoubleIntegrator", 6, 4, 1.4, 3), ("SingleIntegrator", 6, 3, 1.4, 3), ("DubinsCar", 6, 3, 1.6, 3),
         ("LinearDrone", 6, 3, 1.0, 2), ("DoubleIntegrator", 64, 4, 3.2, 6), ("LinearDrone", 32, 3, 1.7, 3)]


KINK_DELTA = 1e-4     # fp32 / 3xTF32 / folded-weight rounding moves an O(10) pre-activation by up to ~1e-5


class _ShiftedReLU(torch.autograd.Function):
    """relu(x) whose derivative is taken as 1[x > delta]: the forward value is the ordinary ReLU."""

    @staticmethod
    def forward(ctx, x, delta):
        ctx.save_for_backward(x)
        ctx.delta = delta
        return x.clamp_min(0)

    @staticmethod
    def backward(ctx, g):
        (x,) = ctx.saved_tensors
        # an exactly-zero pre-activation (masked / padded rows) is not a rounding tie: it keeps derivative 0
        return g * ((x > ctx.delta) & (x != 0)).to(g.dtype), None


class shifted_relu_derivative:
    """Context manager: every torch.relu of the oracle differentiates as 1[x > delta] (forward unchanged)."""

    def __init__(self, delta):
        self.delta = delta

    def __enter__(self):
        self._orig = torch.relu
        torch.relu = lambda x: _ShiftedReLU.apply(x, self.delta)

    def __exit__(self, *exc):
        torch.relu = self._orig
        return False


def _setup(env_id, N, B, area, n_obs, seed=21, pretrained=True):
    agent, goal, obs = random_scene(env_id, N, B, area, n_obs, seed, vel_scale=0.45)
    env = product_env(env_id, N, area, n_obs)
    env.edge_cap_per_agent = 64
    algo = product_algo(env, env_id if pretrained else None, seed=3)
    pobs = product_obstacles(env_id, obs)
    graph = env.get_graph(torch.from_numpy(agent).cuda(), torch.from_numpy(goal).cuda(), pobs)
    rng = np.random.default_rng(seed)
    unsafe = env.unsafe_mask(graph)
    safe = (~unsafe) & torch.from_numpy(rng.uniform(size=(B, N)) < 0.6).cuda()      # some agents unlabelled
    u_qp = env.u_ref(graph) + torch.from_numpy(rng.normal(0, 0.1, size=(B, N, env.action_dim)).astype(np.float32)).cuda()
    return env, algo, graph, pobs, agent, goal, safe, unsafe, u_qp


@pytest.mark.parametrize("env_id,N,B,area,n_obs", CASES)
@pytest.mark.parametrize("pretrained", [True, False])
def test_gradients_match_oracle_autograd(env_id, N, B, area, n_obs, pretrained, gemm_path):
    from gcbfplus_b200.algo.train import read_info, train_minibatch
    from oracle.algo import gcbf_plus_loss
    from oracle.nn import to_torch
    env, algo, graph, pobs, agent, goal, safe, unsafe, u_qp = _setup(env_id, N, B, area, n_obs, pretrained=pretrained)
    # exercise every loss term with comparable weights
    algo.loss_action_coef, algo.loss_h_dot_coef, algo.eps = 0.05, 0.3, 0.02
    ts = train_minibatch(algo, graph, safe, unsafe, u_qp, apply=False)
    torch.cuda.synchronize()
    graph.check_overflow()
    info = read_info(algo)
    # ---- oracle: float64 autograd of the restated loss; float32 evaluated lazily for ReLU-kink ties (below)
    packed = pobs.packed.cpu().numpy()

    def oracle_grads(dt):
        oenv = oracle_env(env_id, N, area, n_obs, dtype=dt)
        cp = to_torch(algo.cbf_params.to_tree(), dt, requires_grad=True)
        ap = to_torch(algo.actor_net_params.to_tree(), dt, requires_grad=True)
        graphs = [oenv.sparsify(oenv.get_graph(torch.from_numpy(agent[g]).to(dt), torch.from_numpy(goal[g]).to(dt),
                                               oracle_obstacles(packed[g], dt))) for g in range(B)]
        total, oinfo = gcbf_plus_loss(oenv, cp, ap, graphs, safe.cpu(), unsafe.cpu(), u_qp.cpu().to(dt), alpha=algo.alpha,
                                      eps=algo.eps, coef_action=algo.loss_action_coef, coef_unsafe=algo.loss_unsafe_coef,
                                      coef_safe=algo.loss_safe_coef, coef_h_dot=algo.loss_h_dot_coef)
        names_c, names_a = list(cp), list(ap)
        gs = torch.autograd.grad(total, [cp[k] for k in names_c] + [ap[k] for k in names_a], allow_unused=True)
        gs = [g.double() if g is not None else None for g in gs]
        return oinfo, names_c, names_a, gs

    oinfo, names_c, names_a, gs = oracle_grads(torch.float64)
    for k in ("loss/action", "loss/unsafe", "loss/safe", "loss/h_dot", "loss/total", "acc/unsafe", "acc/safe",
              "acc/h_dot", "acc/unsafe_data_ratio"):
        assert abs(info[k] - float(oinfo[k])) <= 2e-5 * max(1.0, abs(float(oinfo[k]))), (k, info[k], float(oinfo[k]))
    from gcbfplus_b200.algo.params import NetParams
    any_nonzero = False
    env_lo = env_hi = None      # kink envelope of the float64 oracle, computed only if a tensor disagrees with it
    n_kink = 0
    for net, names, lo, flat in (("cbf", names_c, 0, ts.grad_cbf), ("actor", names_a, len(names_c), ts.grad_act)):
        grads = gs[lo: lo + len(names)]
        proto = algo.cbf_params if net == "cbf" else algo.actor_net_params
        tmp = NetParams(proto.edge_dim, proto.out_dim, proto.kind, device="cuda")
        tmp.flat.copy_(flat)
        got = to_torch(tmp.to_tree(), torch.float64)
        gmax = max(float(g.abs().max()) for g in grads if g is not None)
        any_nonzero = any_nonzero or gmax > 0      # a converged pretrained CBF can have exactly zero loss terms
        for i, k in enumerate(names):
            want = grads[i] if grads[i] is not None else torch.zeros_like(got[k])
            err = float((got[k] - want).abs().max())
            scale = max(float(want.abs().max()), 1e-3 * gmax)
            # 2e-4 of the tensor's own magnitude + 1e-5 of the network's largest gradient entry (fp32 / 3xTF32
            # accumulation noise of a tensor whose entries are small differences of large per-edge terms; measured
            # 5.9e-8 on a bias gradient of magnitude 3.7e-5 next to a largest entry of 1.3e-2)
            tol = 2e-4 * scale + 1e-5 * gmax + 1e-9
            if err <= tol:
                continue
            # ReLU kinks: with ~1e6 hidden units per pass (N = 64: 2 700 edges x 256 x 3 passes) the PRETRAINED networks
            # have a few pre-activations within rounding of 0, where two evaluations of the SAME loss that round
            # differently (float64 oracle, float32 oracle, the layer-by-layer CUDA step, the folded CUDA step) take
            # different one-sided derivatives.  Measured: float64 and float32 oracle differ by 3.2e-3 on the CBF's first
            # layer (one unit); the folded step additionally flips ONE unit of the policy head's first layer (one column
            # of PolicyHead/Dense_0 off by 1e-4, 2.6e-4 on its bias entry), which reaches every upstream actor tensor at
            # 1e-5 .. 7e-4.  Randomly initialised networks have no such ties and must meet `tol` outright (asserted
            # below); a pretrained tensor that misses float64 must stay inside the oracle's own kink envelope: the float64
            # gradient re-evaluated with every ReLU derivative taken as 1[x > +d] and as 1[x > -d] (forward values
            # unchanged, exact zeros excluded), d = KINK_DELTA -- entries no near-zero unit feeds keep `tol`.
            assert pretrained, (net, k, err, tol, "a randomly initialised network has no ReLU ties: strict tolerance")
            if env_lo is None:
                with shifted_relu_derivative(+KINK_DELTA):
                    env_hi = oracle_grads(torch.float64)[3]
                with shifted_relu_derivative(-KINK_DELTA):
                    env_lo = oracle_grads(torch.float64)[3]
            zero = torch.zeros_like(got[k])
            g_hi = env_hi[lo + i] if env_hi[lo + i] is not None else zero
            g_lo = env_lo[lo + i] if env_lo[lo + i] is not None else zero
            slack = 3.0 * ((g_hi - want).abs() + (g_lo - want).abs())
            dev = (got[k] - want).abs()
            excess = float((dev - slack).max())
            assert excess <= tol, (net, k, err, excess, scale)
            n_kink += 1
    assert any_nonzero
    assert n_kink == 0 or pretrained


def test_clip_adamw_and_polyak_match_oracle():
    """Optimizer kernels in isolation: the oracle's float64 clip + AdamW is fed the SAME gradients
    (Adam's m/sqrt(v) is sign-like for near-zero entries, so end-to-end comparison through
    independently rounded gradients is ill-conditioned there)."""
    from gcbfplus_b200.algo.params import NetParams
    from gcbfplus_b200.algo.train import apply_gradients, read_info, train_minibatch, update_tgt
    from oracle.algo import AdamW, compute_norm_and_clip
    from oracle.nn import to_torch
    env_id, N, B, area, n_obs = "DoubleIntegrator", 6, 4, 1.4, 3
    env, algo, graph, pobs, agent, goal, safe, unsafe, u_qp = _setup(env_id, N, B, area, n_obs)
    algo.loss_action_coef, algo.loss_h_dot_coef = 0.05, 0.3
    algo.lr_cbf = algo.lr_actor = 1e-3
    cp = to_torch(algo.cbf_params.to_tree(), torch.float64)
    ap = to_torch(algo.actor_net_params.to_tree(), torch.float64)
    tgt0 = algo.cbf_tgt_params.flat.clone()
    oc, oa = AdamW(cp, lr=1e-3), AdamW(ap, lr=1e-3)

    def tree_of(flat, proto):
        tmp = NetParams(proto.edge_dim, proto.out_dim, proto.kind, device="cuda")
        tmp.flat.copy_(flat)
        return to_torch(tmp.to_tree(), torch.float64)

    for it in range(3):                                            # 3 optimizer steps: bias correction, moments
        ts = train_minibatch(algo, graph, safe, unsafe, u_qp, apply=False)
        gc, ga = tree_of(ts.grad_cbf, algo.cbf_params), tree_of(ts.grad_act, algo.actor_net_params)
        apply_gradients(algo, ts)
        gcc, nc = compute_norm_and_clip(gc, algo.max_grad_norm)
        gac, na = compute_norm_and_clip(ga, algo.max_grad_norm)
        cp, ap = oc.step(cp, gcc), oa.step(ap, gac)
        info = read_info(algo)
        assert abs(info["grad_norm/cbf"] - float(nc)) <= 1e-5 * float(nc)
        assert abs(info["grad_norm/actor"] - float(na)) <= 1e-5 * float(na)
        got_c = to_torch(algo.cbf_params.to_tree(), torch.float64)
        got_a = to_torch(algo.actor_net_params.to_tree(), torch.float64)
        for got, want in ((got_c, cp), (got_a, ap)):
            for k in want:
                assert float((got[k] - want[k]).abs().max()) <= 2e-6, (it, k)   # updates are O(1e-3)
        cp = {k: v.float().double() for k, v in got_c.items()}      # keep the two in lock-step (fp32 storage)
        ap = {k: v.float().double() for k, v in got_a.items()}
    assert int(algo._trainer_state.step_cbf.item()) == 3
    update_tgt(algo, 0.5)
    torch.testing.assert_close(algo.cbf_tgt_params.flat, 0.5 * algo.cbf_params.flat + 0.5 * tgt0)


def test_apply_if_finite_skips_update():
    from gcbfplus_b200.algo.train import apply_gradients, train_minibatch
    env, algo, graph, pobs, agent, goal, safe, unsafe, u_qp = _setup("DoubleIntegrator", 6, 2, 1.4, 2)
    ts = train_minibatch(algo, graph, safe, unsafe, u_qp, apply=False)
    before = algo.cbf_params.flat.clone()
    ts.grad_cbf[5] = float("nan")
    apply_gradients(algo, ts)
    torch.cuda.synchronize()
    assert torch.equal(before, algo.cbf_params.flat) and int(ts.step_cbf.item()) == 0
    assert int(ts.step_act.item()) == 1


def test_gemm_kernels_match_torch_fp32():
    """Numerics of the GEMM building blocks vs plain PyTorch fp32 (allow_tf32 off)."""
    import ctypes as C
    from gcbfplus_b200 import _lib
    lib = _lib.load()
    torch.backends.cuda.matmul.allow_tf32 = False
    st = torch.cuda.current_stream().cuda_stream
    g = torch.Generator(device="cuda").manual_seed(0)
    for (M, K, N) in [(1, 128, 128), (300, 256, 256), (1000, 128, 256), (4097, 256, 128)]:
        A = torch.randn(M, K, device="cuda", generator=g)
        W = torch.randn(K, N, device="cuda", generator=g) * 0.1
        b = torch.randn(N, device="cuda", generator=g)
        b2 = torch.randn(N, device="cuda", generator=g)
        out = torch.empty(M, N, device="cuda")
        mcount = torch.tensor([M], dtype=torch.int32, device="cuda")
        _lib.check(lib.gcbf_gemm_nn(1, 0, A.data_ptr(), W.data_ptr(), b.data_ptr(), b2.data_ptr(), out.data_ptr(), None,
                                    mcount.data_ptr(), 0, M, K, N, st))
        torch.testing.assert_close(out, torch.relu(A @ W + b + b2), atol=2e-4, rtol=1e-5)
        aux = torch.randn(M, N, device="cuda", generator=g)
        acc = torch.randn(M, N, device="cuda", generator=g)
        want = acc + (A @ W) * (aux > 0)
        _lib.check(lib.gcbf_gemm_nn(3, 1, A.data_ptr(), W.data_ptr(), None, None, acc.data_ptr(), aux.data_ptr(), None,
                                    M, M, K, N, st))
        torch.testing.assert_close(acc, want, atol=2e-4, rtol=1e-5)
    for (M, K1, N) in [(5, 128, 128), (777, 256, 128), (20000, 128, 256)]:
        X = torch.randn(M, K1, device="cuda", generator=g)
        dY = torch.randn(M, N, device="cuda", generator=g)
        w = (torch.rand(64, device="cuda", generator=g) > 0.3).float()
        r2a = torch.randint(0, 64, (M,), device="cuda", generator=g, dtype=torch.int32)
        Cw = torch.zeros(K1, N, device="cuda")
        db = torch.zeros(N, device="cuda")
        _lib.check(lib.gcbf_gemm_tn(X.data_ptr(), K1, dY.data_ptr(), Cw.data_ptr(), w.data_ptr(), r2a.data_ptr(), None, M,
                                    M, K1, N, 64, st))
        _lib.check(lib.gcbf_colsum(dY.data_ptr(), db.data_ptr(), w.data_ptr(), r2a.data_ptr(), None, M, M, N, 64, st))
        wd = dY * w[r2a.long()][:, None]
        torch.testing.assert_close(Cw, X.T @ wd, atol=1e-3 * (M ** 0.5) / 10 + 1e-4, rtol=1e-4)
        torch.testing.assert_close(db, wd.sum(0), atol=1e-3 * (M ** 0.5) / 10 + 1e-4, rtol=1e-4)


def test_tensor_core_gemm_matches_float64():
    """wgmma 3xTF32 GEMM (gemm_tc.cuh) vs a float64 reference: fp32-class accuracy
    (<= 2e-6 of |A||B|; single-pass TF32 would be ~5e-4), all epilogues, ragged M, device row count."""
    from gcbfplus_b200 import _lib
    lib = _lib.load()
    st = torch.cuda.current_stream().cuda_stream
    g = torch.Generator(device="cuda").manual_seed(0)
    for (M, K, N, cap, epi, accum) in [(1, 32, 128, 128, 0, 0), (128, 128, 128, 128, 0, 0), (300, 256, 256, 300, 1, 0),
                                       (1000, 128, 256, 1024, 2, 0), (4097, 256, 128, 5000, 3, 0),
                                       (14012, 256, 256, 16000, 3, 1), (777, 256, 256, 777, 2, 1)]:
        A = torch.randn(cap, K, device="cuda", generator=g)
        W = torch.randn(K, N, device="cuda", generator=g) * 0.1
        Bt = W.t().contiguous()
        Bh, Bl = torch.empty_like(Bt), torch.empty_like(Bt)
        _lib.check(lib.gcbf_split_tf32(Bt.data_ptr(), Bh.data_ptr(), Bl.data_ptr(), Bt.numel(), st))
        assert float((Bh + Bl - Bt).abs().max()) <= 2 ** -23 * float(Bt.abs().max())
        b = torch.randn(N, device="cuda", generator=g)
        b2 = torch.randn(N, device="cuda", generator=g)
        aux = torch.randn(cap, N, device="cuda", generator=g)
        out = torch.full((cap, N), 7.0, device="cuda")
        mc = torch.tensor([M], dtype=torch.int32, device="cuda")
        _lib.check(lib.gcbf_gemm_tc(epi, accum, A.data_ptr(), Bh.data_ptr(), Bl.data_ptr(), b.data_ptr(), b2.data_ptr(), out.data_ptr(),
                                    aux.data_ptr(), mc.data_ptr(), 0, cap, K, N, 0, st))
        ref = A[:M].double() @ W.double()
        if epi in (0, 1):
            ref = ref + b.double() + b2.double()
        if epi == 1:
            ref = torch.relu(ref)
        if epi == 3:
            ref = ref * (aux[:M] > 0)
        if accum:
            ref = ref + 7.0
        scale = float((A[:M].abs().double() @ W.abs().double()).max())
        err = float((out[:M].double() - ref).abs().max())
        assert err <= 2e-6 * scale, (M, K, N, epi, accum, err, scale)
        assert bool((out[M:] == 7.0).all())                     # rows >= M untouched


def test_tensor_core_relu_dotn_epilogue_matches_float64():
    """EPI_RELU_DOTN (output-layer partial sums per 128-wide column tile) of the wgmma GEMM vs float64, ragged M from a
    device counter; rows >= M untouched."""
    from gcbfplus_b200 import _lib
    lib = _lib.load()
    st = torch.cuda.current_stream().cuda_stream
    g = torch.Generator(device="cuda").manual_seed(1)
    for (M, K, N, cap, ndot) in [(1, 256, 256, 128, 2), (777, 256, 256, 800, 3), (9000, 256, 256, 9000, 4)]:
        A = torch.randn(cap, K, device="cuda", generator=g)
        W = torch.randn(K, N, device="cuda", generator=g) * 0.1
        Bt = W.t().contiguous()
        Bh, Bl = torch.empty_like(Bt), torch.empty_like(Bt)
        _lib.check(lib.gcbf_split_tf32(Bt.data_ptr(), Bh.data_ptr(), Bl.data_ptr(), Bt.numel(), st))
        b = torch.randn(N, device="cuda", generator=g)
        b2 = torch.randn(1, device="cuda", generator=g)
        aux = torch.randn(N * ndot, device="cuda", generator=g)
        parts = N // 128
        out = torch.full((parts * cap * 4,), 7.0, device="cuda")
        mc = torch.tensor([M], dtype=torch.int32, device="cuda")
        _lib.check(lib.gcbf_gemm_tc(5, 0, A.data_ptr(), Bh.data_ptr(), Bl.data_ptr(), b.data_ptr(), b2.data_ptr(),
                                    out.data_ptr(), aux.data_ptr(), mc.data_ptr(), 0, cap, K, N, ndot, st))
        h = torch.relu(A[:M].double() @ W.double() + b.double())
        hs = (A[:M].abs().double() @ W.abs().double() + b.abs().double())      # |pre-activation| bound per entry
        o = out.view(parts, cap, 4)
        av = aux.view(N, ndot).double()
        for p in range(parts):
            cols = slice(128 * p, 128 * (p + 1))
            ref = h[:, cols] @ av[cols]
            tol = 1e-5 * float((hs[:, cols] @ av[cols].abs()).max())
            assert float((o[p, :M, :ndot].double() - ref).abs().max()) <= tol, (M, K, N, p)
            assert bool((o[p, :M, ndot:] == 0).all())
            assert bool((o[p, M:] == 7.0).all())


def test_tensor_core_gemm_rejects_unassigned_epilogue():
    """Epilogue 4 is unassigned (the gate logit is only produced by the chained edge kernel): gcbf_gemm_tc returns an
    error status with an error string and writes nothing."""
    from gcbfplus_b200 import _lib
    lib = _lib.load()
    st = torch.cuda.current_stream().cuda_stream
    g = torch.Generator(device="cuda").manual_seed(1)
    A = torch.randn(128, 128, device="cuda", generator=g)
    Bh = torch.zeros(128, 128, device="cuda")
    b = torch.randn(128, device="cuda", generator=g)
    out = torch.full((128,), 7.0, device="cuda")
    with pytest.raises(RuntimeError, match="bad epilogue"):
        _lib.check(lib.gcbf_gemm_tc(4, 0, A.data_ptr(), Bh.data_ptr(), Bh.data_ptr(), b.data_ptr(), b.data_ptr(),
                                    out.data_ptr(), b.data_ptr(), None, 128, 128, 128, 128, 0, st))
    torch.cuda.synchronize()
    assert bool((out == 7.0).all())


def test_tensor_core_weight_gradient_matches_float64():
    """gcbf_gemm_tn_tc (weight gradient C += X^T diag(w) dY with the bias-gradient column sums of the same pass) vs
    float64: N = 128 / 256, ragged M from a device counter with NaN in the rows >= M, a row stride wider than K1, several
    M-splits per column tile, per-row weights through row2agent, cs1 / cs2 accumulated onto their previous contents."""
    from gcbfplus_b200 import _lib
    lib = _lib.load()
    st = torch.cuda.current_stream().cuda_stream
    g = torch.Generator(device="cuda").manual_seed(2)
    n_ag = 64
    for (M, cap, K1, ldx, N) in [(1, 32, 128, 128, 128), (5, 40, 128, 132, 256), (777, 800, 256, 256, 128),
                                 (1000, 1000, 128, 256, 256), (20011, 20480, 256, 260, 256), (4100, 4224, 384, 384, 128)]:
        X = torch.randn(cap, ldx, device="cuda", generator=g)
        dY = torch.randn(cap, N, device="cuda", generator=g)
        X[M:] = float("nan")
        dY[M:] = float("nan")
        w = torch.rand(n_ag, device="cuda", generator=g) * (torch.rand(n_ag, device="cuda", generator=g) > 0.3)
        r2a = torch.randint(0, n_ag, (cap,), device="cuda", generator=g, dtype=torch.int32)
        C0 = torch.randn(K1, N, device="cuda", generator=g)
        Cw = C0.clone()
        cs1 = torch.zeros(N, device="cuda")
        cs2 = torch.randn(N, device="cuda", generator=g)
        cs2_0 = cs2.clone()
        mc = torch.tensor([M], dtype=torch.int32, device="cuda")
        _lib.check(lib.gcbf_gemm_tn_tc(X.data_ptr(), ldx, dY.data_ptr(), Cw.data_ptr(), w.data_ptr(), r2a.data_ptr(),
                                       mc.data_ptr(), 0, cap, K1, N, n_ag, cs1.data_ptr(), cs2.data_ptr(), st))
        wd = dY[:M].double() * w[r2a[:M].long()].double()[:, None]
        x = X[:M, :K1].double()
        ref = C0.double() + x.t() @ wd
        scale = float((x.abs().t() @ wd.abs()).max()) + float(C0.abs().max())
        assert bool(torch.isfinite(Cw).all())
        assert float((Cw.double() - ref).abs().max()) <= 1e-5 * scale, (M, K1, N)
        cref = wd.sum(0)
        ctol = 1e-5 * float(wd.abs().sum(0).max()) + 1e-6
        assert float((cs1.double() - cref).abs().max()) <= ctol, (M, N)
        assert float((cs2.double() - cs2_0.double() - cref).abs().max()) <= ctol, (M, N)
