"""The fused SGD-momentum / LARS sweep (esvit_b200.optim.FusedSGDEMA: esvit_lars_sums_multi + esvit_sgd_ema_multi)
against the reference's --optimizer sgd / lars step tail (oracle/optim.py, pinned to the reference by
tests/test_optim_oracle.py), its state_dict interchange with the reference's optimiser objects, and the training step
built with make_step(optimizer_type=sgd | lars)."""
import copy

import pytest
import torch
import torch.nn as nn

from helpers import assert_close

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16


def _dev():
    return torch.device("cuda:0")


class Toy(nn.Module):
    """the AdamW sweep test's toy module plus the LARS corner cases: a zero-valued 2-D weight (||p|| = 0) and a 2-D
    `.bias` of group 1 whose gradient is zero (wd 0, so ||d|| = 0); both take q = 1"""

    def __init__(self):
        super().__init__()
        self.a = nn.Linear(33, 65)
        self.norm = nn.LayerNorm(65)
        self.z = nn.Linear(65, 7, bias=False)
        self.tok = nn.Module()
        self.tok.bias = nn.Parameter(torch.randn(3, 5))
        self.last_layer = nn.Linear(65, 130, bias=False)
        self.g = nn.Parameter(torch.ones(130, 1), requires_grad=False)


def _toy_pair(seed=7):
    torch.manual_seed(seed)
    ref_s = Toy()
    with torch.no_grad():
        ref_s.z.weight.zero_()
    ref_t = Toy()
    ref_t.load_state_dict(ref_s.state_dict())
    d = _dev()
    s, t = Toy().to(d), Toy().to(d)
    s.load_state_dict(ref_s.state_dict())
    t.load_state_dict(ref_s.state_dict())
    for p_ in list(ref_t.parameters()) + list(t.parameters()):
        p_.requires_grad = False
    return ref_s, ref_t, s, t


def _grads(module, it, g):
    return {n: (torch.zeros(p_.shape) if n == "tok.bias" else
                torch.randn(p_.shape, generator=g) * (20.0 if it % 2 == 0 else 0.05))
            for n, p_ in module.named_parameters() if p_.requires_grad}


STEPS = [(1e-1, 0.04, 0.996, True), (2e-1, 0.05, 0.997, True), (5e-2, 0.1, 0.99, False)]


@pytest.mark.parametrize("misaligned", [False, True])
@pytest.mark.parametrize("kind", ["sgd", "lars"])
def test_fused_sgd_lars_matches_reference_sequence(kind, misaligned):
    """esvit_sgd_ema_multi == clip_gradients -> cancel last_layer grads -> torch.optim.SGD / LARS step -> EMA loop over 3
    steps with changing lr / wd / momentum, the skip flag on then off.  misaligned: the gradients are views of ONE flat
    bucket at odd element offsets -> the scalar paths of both kernels must update every element."""
    from esvit_b200.optim import FusedSGDEMA
    from oracle import optim as O

    ref_s, ref_t, s, t = _toy_pair()
    d = _dev()
    ropt = O.make_optimizer(kind, ref_s)
    fopt = FusedSGDEMA(s, t, lars=(kind == "lars"), clip_grad=3.0)
    init_tok = s.tok.bias.detach().clone()
    g = torch.Generator().manual_seed(8)
    for it, (lr, wd, mom, skip) in enumerate(STEPS):
        grads = _grads(ref_s, it, g)
        if misaligned:
            flat = torch.zeros(sum(g_.numel() + 8 for g_ in grads.values()) + 8, device=d)
            off = 1
            for n, p_ in s.named_parameters():
                if n in grads:
                    view = flat[off:off + p_.numel()].view(p_.shape)
                    view.copy_(grads[n])
                    assert view.data_ptr() % 16 != 0
                    p_.grad = view
                    off = ((off + p_.numel() + 3) // 4) * 4 + 1  # every view starts 4 bytes past a 16-byte boundary
                else:
                    p_.grad = None
        else:
            for n, p_ in s.named_parameters():
                p_.grad = grads[n].clone().to(d) if n in grads else None
        O.train_step_tail(ref_s, ref_t, ropt, grads, lr, wd, mom, skip, 3.0)
        fopt.set_hyper(lr, wd, mom)
        fopt.set_skip_last_layer(skip)
        t_before = [p_.detach().clone() for p_ in t.parameters()]
        fopt.step()
        for (n, a), b in zip(s.named_parameters(), ref_s.parameters()):
            assert_close(a, b, 2e-6, f"{kind} param {n} step {it}")
        for (n, a), b in zip(t.named_parameters(), ref_t.parameters()):
            assert_close(a, b, 2e-6, f"{kind} teacher {n} step {it}")
        for k0, k1, q in zip(t_before, t.parameters(), s.parameters()):  # EMA bit-exact w.r.t. OUR updated student
            assert torch.equal(k1, k0.mul_(mom).add_((1 - mom) * q.detach()))
        rbuf = O.buffers(ropt, ref_s)
        for i, (n, p_) in enumerate(s.named_parameters()):
            if n in rbuf:  # state[:, 0] marks "has a buffer"
                assert float(fopt.state[i, 0]) > 0, n
                if float(rbuf[n].norm()) > 0:
                    assert_close(fopt.momentum_buffer[i], rbuf[n], 2e-6, f"{kind} buffer {n} step {it}")
                else:
                    assert float(fopt.momentum_buffer[i].abs().max()) == 0, n
            else:
                assert float(fopt.state[i, 0]) == 0, n
        assert torch.equal(s.tok.bias.detach(), init_tok)  # zero gradient, wd 0: q = 1 and no movement
        norms = fopt.grad_norms().cpu()
        for (n, p_), nr in zip(s.named_parameters(), norms):
            if n in grads:
                assert abs(float(nr) - float(grads[n].double().norm())) <= 1e-5 * float(grads[n].norm()) + 1e-12, n


@pytest.mark.parametrize("kind", ["sgd", "lars"])
def test_fused_sgd_lars_writes_bf16_shadows(kind):
    """after a step every registered bf16 shadow of the student and the teacher is the bf16 cast of its parameter"""
    from esvit_b200.optim import FusedSGDEMA

    _, _, s, t = _toy_pair(3)
    fopt = FusedSGDEMA(s, t, lars=(kind == "lars"))
    fopt.set_hyper(0.1, 0.04, 0.996)
    fopt.set_skip_last_layer(False)
    g = torch.Generator().manual_seed(4)
    for it in range(2):
        grads = _grads(s, it, g)
        for n, p_ in s.named_parameters():
            p_.grad = grads[n].to(_dev()) if n in grads else None
        fopt.step()
    nsh = 0
    for params, shadows in ((fopt.params, fopt.shadow_p), (fopt.teacher_params, fopt.shadow_k)):
        for p_, sh in zip(params, shadows):
            if sh is not None:
                nsh += 1
                assert torch.equal(sh, p_.detach().to(BF16))
    assert nsh >= 8  # a.weight, a.bias, z.weight, tok.bias of each network


def _stepped_fused(kind, skip_last):
    from esvit_b200.optim import FusedSGDEMA

    torch.manual_seed(3)
    s, t = Toy().to(_dev()), Toy().to(_dev())
    for p_ in t.parameters():
        p_.requires_grad = False
    fopt = FusedSGDEMA(s, t, lars=(kind == "lars"), clip_grad=3.0)
    fopt.set_hyper(1e-2, 0.04, 0.996)
    fopt.set_skip_last_layer(skip_last)
    for _ in range(2):
        for n, p_ in s.named_parameters():
            p_.grad = torch.randn_like(p_) if p_.requires_grad else None
        fopt.step()
    return s, t, fopt


@pytest.mark.parametrize("kind", ["sgd", "lars"])
def test_fused_sgd_lars_state_dict_interchanges_with_reference_optimizers(kind):
    """FusedSGDEMA.state_dict() uses the reference's optimiser layout over utils.get_params_groups (torch.optim.SGD's
    momentum_buffer, utils.LARS's mu; one entry per stepped tensor): the reference's optimiser loads it, and a fresh
    fused optimiser resumes from the reference optimiser's state_dict."""
    from esvit_b200 import utils
    from esvit_b200.optim import FusedSGDEMA
    from oracle import optim as O

    s, t, fopt = _stepped_fused(kind, skip_last=True)
    sd = fopt.state_dict()
    key = "mu" if kind == "lars" else "momentum_buffer"
    ropt = (torch.optim.SGD(utils.get_params_groups(s), lr=0, momentum=0.9) if kind == "sgd"
            else O.LARS(utils.get_params_groups(s)))
    ropt.load_state_dict(sd)
    rparams = [p_ for g_ in ropt.param_groups for p_ in g_["params"]]
    reg, noreg = fopt._torch_order()
    names = fopt.names
    for k, i in enumerate(reg + noreg):
        assert rparams[k] is fopt.params[i]
        if "last_layer" in names[i]:  # cancelled on both steps: no buffer, as in the reference
            assert rparams[k] not in ropt.state
        else:
            assert torch.equal(ropt.state[rparams[k]][key], fopt.momentum_buffer[i])
    assert ropt.param_groups[0]["weight_decay"] == pytest.approx(0.04) and ropt.param_groups[1]["weight_decay"] == 0
    # and back: a fresh fused optimiser resumes from the reference optimiser's state
    f2 = FusedSGDEMA(s, t, lars=(kind == "lars"), clip_grad=3.0)
    f2.load_state_dict(ropt.state_dict())
    for a, b in zip(f2.momentum_buffer, fopt.momentum_buffer):
        assert torch.equal(a, b)
    assert torch.equal(f2.state[:, 0] > 0, fopt.state[:, 0] > 0)
    # both resume identically: one more step of the reference optimiser and of a fused one loaded from its state
    rsd = copy.deepcopy(ropt.state_dict())
    s2 = Toy().to(_dev())
    s2.load_state_dict(s.state_dict())
    grads = {n: torch.randn_like(p_) for n, p_ in s.named_parameters() if p_.requires_grad}
    ropt.param_groups[0]["lr"] = ropt.param_groups[1]["lr"] = 1e-2
    ropt.param_groups[0]["weight_decay"] = 0.04
    for n, p_ in s.named_parameters():
        p_.grad = grads[n].clone() if n in grads else None
    ropt.step()  # no clip on either side (clip_grad=0.0 below)
    after_ref = {n: p_.detach().clone() for n, p_ in s.named_parameters()}
    s.load_state_dict(s2.state_dict())
    f3 = FusedSGDEMA(s, None, lars=(kind == "lars"), clip_grad=0.0)
    f3.load_state_dict(rsd)
    f3.set_hyper(1e-2, 0.04, 0.996)
    f3.set_skip_last_layer(False)
    for n, p_ in s.named_parameters():
        p_.grad = grads[n].clone() if n in grads else None
    f3.step()
    for n, p_ in s.named_parameters():
        assert_close(p_, after_ref[n], 2e-6, f"{kind} resumed {n}")


def _make(kind, optimizer="fused", cuda_graph=False):
    """Swin-T W7 step with non-zero biases, LayerNorm affines and bias tables: SGD moves a zero-initialised parameter
    by lr * g alone, so its relative difference would be the relative fp32-atomic noise of its gradient (the patch
    embedding LN beta's sums cancel heavily), not a measure of the step"""
    from esvit_b200 import engine
    step, student, teacher, loss = engine.make_step(arch="swin_tiny_w7", out_dim=4096, ncrops=4, dense=True,
                                                    device="cuda:0", drop_path=0.0, optimizer=optimizer,
                                                    optimizer_type=kind, cuda_graph=cuda_graph, seed=5)
    g = torch.Generator().manual_seed(11)
    with torch.no_grad():
        for n, p_ in student.named_parameters():
            if n.endswith(".bias") or p_.dim() == 1 or "relative_position_bias_table" in n:
                p_.add_(torch.randn(p_.shape, generator=g).to(p_.device) * 0.1)
    teacher.load_state_dict(student.state_dict())
    return step, student, teacher, loss


def _crops(B=2, nlocal=2):
    g = torch.Generator().manual_seed(1)
    crops = [torch.randn(B, 3, 224, 224, generator=g) for _ in range(2)]
    crops += [torch.randn(B, 3, 96, 96, generator=g) for _ in range(nlocal)]
    return [c.cuda() for c in crops]


@pytest.mark.parametrize("kind", ["sgd", "lars"])
def test_sgd_lars_cuda_graph_step_equals_eager_step(kind):
    """the graph-captured step with the fused SGD / LARS sweep computes what its eager body computes, under the gate
    of the AdamW graph test (2e-3: fp32 atomic-order noise of the small-parameter gradients)"""
    from esvit_b200.optim import FusedSGDEMA

    stepE, sE, _, lE = _make(kind)
    stepG, sG, _, lG = _make(kind, cuda_graph=True)
    assert isinstance(stepG.opt, FusedSGDEMA) and stepG.opt.lars == (kind == "lars") and stepG.use_cuda_graph
    crops = _crops()
    le, lg = [], []
    for it in range(6):  # 3 eager warm-up calls + capture + 2 replays on the graph side
        lr = 1e-2 * (1 + 0.1 * it)
        le.append(float(stepE(crops, 1, lr, 0.04, 0.996)))
        lg.append(float(stepG(crops, 1, lr, 0.04, 0.996)))
    assert len(stepG._graphs) == 1
    for a, b in zip(le, lg):
        assert abs(a - b) < 2e-3 * abs(a), (le, lg)
    for (n, a), b in zip(sE.named_parameters(), sG.parameters()):
        assert_close(b, a, 2e-3, n)
    assert_close(lG.center, lE.center, 1e-3, "center")


def test_fused_sgd_step_equals_torch_sgd_step():
    """make_step(optimizer_type="sgd"): the fused sweep and the reference's own torch.optim.SGD step agree within the
    graph test's gate after 2 steps"""
    stepF, sF, tF, _ = _make("sgd")
    stepT, sT, tT, _ = _make("sgd", optimizer="torch")
    assert isinstance(stepT.opt, torch.optim.SGD) and not stepT.fused
    crops = _crops()
    lf, lt = [], []
    for it in range(2):
        lf.append(float(stepF(crops, it, 1e-2, 0.04, 0.996)))  # epoch 0: last layer cancelled, epoch 1: stepped
        lt.append(float(stepT(crops, it, 1e-2, 0.04, 0.996)))
    for a, b in zip(lf, lt):
        assert abs(a - b) < 2e-3 * abs(b), (lf, lt)
    for (n, a), b in zip(sF.named_parameters(), sT.parameters()):
        assert_close(a, b, 2e-3, n)
    for (n, a), b in zip(tF.named_parameters(), tT.parameters()):
        assert_close(a, b, 2e-3, "teacher " + n)


def test_make_step_optimizer_type_choices():
    from esvit_b200 import engine
    from esvit_b200.optim import FusedAdamWEMA
    with pytest.raises(ValueError):
        engine.make_step(optimizer="torch", optimizer_type="lars")
    with pytest.raises(ValueError):
        engine.make_step(optimizer_type="adam")
    step = engine.make_step(arch="swin_tiny_w7", out_dim=256, ncrops=4, device="cuda:0")[0]
    assert type(step.opt) is FusedAdamWEMA  # the default is unchanged
