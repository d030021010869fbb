import pytest
import torch

from acco_b200.optim import AdamHyper, ShardedAdamW, adamw_shard_update_
from acco_b200.parallel.schedule import COMMIT_ALL, COMMIT_NONE, LRSchedule, RoundScheduler, get_lr_lambda


def test_matches_torch_adamw():
    torch.manual_seed(0)
    p0 = torch.randn(257)
    ref = p0.clone().requires_grad_(True)
    opt = torch.optim.AdamW([ref], lr=3e-3, betas=(0.9, 0.95), eps=1e-8, weight_decay=0.1)
    mine = ShardedAdamW(p0, lr=3e-3, betas=(0.9, 0.95), eps=1e-8, weight_decay=0.1)
    out = torch.zeros(257)
    for step in range(1, 6):
        g = torch.randn(257)
        ref.grad = g.clone()
        opt.step()
        hp = AdamHyper(lr=3e-3, beta1=0.9, beta2=0.95, eps=1e-8, weight_decay=0.1, step=step, inv_count=0.5, commit=COMMIT_ALL)
        adamw_shard_update_(2 * g, mine.master, mine.exp_avg, mine.exp_avg_sq, mine.stash, out, hp)
        torch.testing.assert_close(mine.master, ref.detach(), rtol=1e-6, atol=1e-7)
        torch.testing.assert_close(out, ref.detach(), rtol=1e-6, atol=1e-7)


def test_tentative_step_does_not_touch_state_and_stash_roundtrip():
    torch.manual_seed(1)
    p0 = torch.randn(64)
    o = ShardedAdamW(p0, lr=1e-2)
    out_t, out_r = torch.zeros(64), torch.zeros(64)
    g_tilde, g = torch.randn(64), torch.randn(64)
    before = (o.master.clone(), o.exp_avg.clone(), o.exp_avg_sq.clone())
    # tentative: consume g~ (count 1), stash it, commit nothing
    adamw_shard_update_(g_tilde, o.master, o.exp_avg, o.exp_avg_sq, o.stash, out_t,
                        AdamHyper(lr=1e-2, step=1, inv_count=1.0, commit=COMMIT_NONE, write_stash=True))
    for a, b in zip(before, (o.master, o.exp_avg, o.exp_avg_sq)):
        assert torch.equal(a, b)
    assert torch.equal(o.stash, g_tilde) and not torch.equal(out_t, p0)
    # real: consume g + stash, count 2  == a single AdamW step on the mean gradient
    adamw_shard_update_(g, o.master, o.exp_avg, o.exp_avg_sq, o.stash, out_r,
                        AdamHyper(lr=1e-2, step=1, inv_count=0.5, commit=COMMIT_ALL, add_stash=True))
    ref = p0.clone().requires_grad_(True)
    topt = torch.optim.AdamW([ref], lr=1e-2)
    ref.grad = (g + g_tilde) / 2
    topt.step()
    torch.testing.assert_close(o.master, ref.detach(), rtol=1e-6, atol=1e-7)


def test_device_scalar_inv_count():
    o = ShardedAdamW(torch.ones(8), lr=1e-1, weight_decay=0.0)
    out = torch.zeros(8)
    adamw_shard_update_(torch.full((8,), 4.0), o.master, o.exp_avg, o.exp_avg_sq, o.stash, out,
                        AdamHyper(lr=1e-1, step=1, inv_count=torch.tensor([0.25]), weight_decay=0.0))
    torch.testing.assert_close(out, torch.full((8,), 0.9), rtol=1e-5, atol=1e-6)   # first Adam step moves by lr


@pytest.mark.parametrize("name", ["cosine", "linear", "constant", "constant_with_warmup"])
def test_lr_lambdas_match_transformers(name):
    transformers = pytest.importorskip("transformers")
    p = torch.nn.Parameter(torch.zeros(1))
    opt = torch.optim.SGD([p], lr=1.0)
    kw = {} if name == "constant" else {"num_warmup_steps": 7}
    if name in ("cosine", "linear"):
        kw["num_training_steps"] = 50
    hf = transformers.get_scheduler(name, optimizer=opt, **kw)
    f = get_lr_lambda(name, 7, 50)
    for k in range(60):
        assert hf.get_last_lr()[0] == pytest.approx(f(k), abs=1e-9), (name, k)
        opt.step()
        hf.step()


def test_lr_units():
    s = RoundScheduler("acco")
    lr = LRSchedule(1.0, "linear", 0, 10, unit="optimizer_step")
    lrg = LRSchedule(1.0, "linear", 0, 10, unit="grads")
    for _ in range(4):
        plan = s.next_plan()
        s.complete(plan, 3)
    # 4 rounds = 2 real steps; each real step counted 3 grads
    assert s.lr_steps == 2 and s.count_grad_tot == 6
    assert lr.lr_at(s) == pytest.approx(0.8) and lrg.lr_at(s) == pytest.approx(0.4)


def test_gemm_reference_layouts_match_torch():
    """CPU path of ops.gemm (the numerics oracle of the wgmma kernel): K-major / MN-major operands, bias, accumulate."""
    import torch
    from acco_b200.ops.gemm import gemm, gemm_nn, gemm_tn, gemm_tt_acc
    torch.manual_seed(0)
    x, w, dy = torch.randn(12, 8), torch.randn(6, 8), torch.randn(12, 6)
    b = torch.randn(6)
    torch.testing.assert_close(gemm_tn(x, w, bias=b), x @ w.t() + b)
    torch.testing.assert_close(gemm_nn(dy, w), dy @ w)
    g = torch.ones(6, 8)
    gemm_tt_acc(dy, x, g)
    torch.testing.assert_close(g, 1 + dy.t() @ x)
    torch.testing.assert_close(gemm(dy, x, a_mn=True, b_mn=True), dy.t() @ x)


def test_linear_autograd_matches_torch_with_grad_accumulation():
    import torch
    from acco_b200.ops import linear
    torch.manual_seed(1)
    x = torch.randn(5, 3, 8, requires_grad=True)
    w = torch.nn.Parameter(torch.randn(6, 8))
    b = torch.nn.Parameter(torch.randn(6))
    w.grad, b.grad = torch.full_like(w, 2.0), torch.full_like(b, -1.0)
    y = linear(x, w, b)
    y.square().sum().backward()
    xr, wr, br = x.detach().clone().requires_grad_(True), w.detach().clone().requires_grad_(True), b.detach().clone().requires_grad_(True)
    torch.nn.functional.linear(xr, wr, br).square().sum().backward()
    torch.testing.assert_close(x.grad, xr.grad)
    torch.testing.assert_close(w.grad, 2.0 + wr.grad)          # accumulated into the existing (arena) gradient
    torch.testing.assert_close(b.grad, -1.0 + br.grad)
