"""GPU: the linear probe (esvit_b200.probe, eval_linear.py's train() / validate_network()) - the cross-entropy kernel and
the fp32-output GEMM against fp64, LinearProbeStep against the reference's trajectory (tests/golden/esvit_probe.pt),
graph replay, ragged batches, checkpoints in both directions with torch.optim.SGD + CosineAnnealingLR, the Swin-T
probe features inside the step, and input validation."""
import os

import pytest
import torch

from oracle import make_golden_probe as MG
from oracle import probe as PR

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "esvit_probe.pt")
U = 2.0 ** -8  # bf16 unit roundoff


@pytest.fixture(scope="module")
def G():
    return MG.load(GOLDEN)


class _Features:
    """a frozen 'backbone' whose images are the features themselves, viewed [B, D, 1, 1]"""

    def forward_return_n_last_blocks(self, x, n, avgpool, depths):
        return x.reshape(x.shape[0], -1)


def _as_images(x):
    return x.cuda().reshape(x.shape[0], -1, 1, 1).contiguous()


def _batches(x, y, B):
    return [(x[r:r + B], y[r:r + B]) for r in range(0, x.shape[0], B)]


def _probe(G, graph=False, seed=None):
    from esvit_b200 import probe
    p = G["params"]
    torch.manual_seed(p["init_seed"] if seed is None else seed)
    clf = probe.LinearClassifier(p["D"], p["C"]).cuda()
    opt = probe.ProbeSGD(clf.parameters(), p["lr"], momentum=0.9, weight_decay=0)
    sched = torch.optim.lr_scheduler.CosineAnnealingLR(opt, p["epochs"], eta_min=0)
    step = probe.LinearProbeStep(_Features(), clf, opt, 4, False, [], use_cuda_graph=graph)
    return clf, opt, sched, step


def _run(G, graph=False, epochs=None):
    """the fixture's epochs through LinearProbeStep -> (classifier, losses [device scalars], per-step (w, b, bufs))"""
    clf, opt, sched, step = _probe(G, graph)
    x, y = G["train"]
    p = G["params"]
    losses, states = [], []
    for _ in range(p["epochs"] if epochs is None else epochs):
        for xb, yb in _batches(x, y, p["batch"]):
            losses.append(step(_as_images(xb), yb))
            sw = opt.sweep
            states.append(tuple(t.detach().clone() for t in (clf.linear.weight, clf.linear.bias,
                                                              sw.momentum_buffer[0], sw.momentum_buffer[1])))
        sched.step()
    return clf, opt, step, losses, states


# ---- esvit_probe_ce against fp64 ----------------------------------------------------------------------------------
def _ce(logits, labels, ld, grad=True):
    from esvit_b200 import _lib
    from esvit_b200.ops import _p, _stream
    B, C = logits.shape
    lg = torch.zeros(B, ld, dtype=torch.float32, device="cuda")
    lg[:, :C] = logits
    lab = labels.cuda()
    d = torch.full((B, ld), float("nan"), dtype=torch.bfloat16, device="cuda") if grad else None
    rl = torch.empty(B, device="cuda")
    rr = torch.empty(B, dtype=torch.int32, device="cuda")
    loss = torch.empty(1, device="cuda")
    acc = torch.zeros(1, dtype=torch.float64, device="cuda")
    cnt = torch.zeros(4, dtype=torch.int64, device="cuda")
    _lib.call("esvit_probe_ce", _p(lg), ld, _p(lab), B, C, _p(d), _p(rl), _p(rr), _p(loss), _p(acc), _p(cnt),
              _stream())
    torch.cuda.synchronize()
    return d, rl, rr, loss, acc, cnt


@pytest.mark.parametrize("B", [8, 13, 128, 256])
@pytest.mark.parametrize("C", [10, 1000])
def test_probe_ce_matches_fp64(B, C):
    g = torch.Generator().manual_seed(B * 7 + C)
    logits = torch.randn(B, C, generator=g) * 3
    labels = torch.randint(0, C, (B,), generator=g)
    labels[::5] = -1  # padding rows
    # exact ties with the target: equal values ahead / behind by index
    for r in range(1, B, 3):
        t = int(labels[r])
        if t >= 0:
            logits[r, (t + 1) % C] = logits[r, t]
            logits[r, (t + C - 1) % C] = logits[r, t]
    ld = -(-C // 8) * 8 + (8 if C == 10 else 0)  # also a row pitch beyond the padded classes
    d, rl, rr, loss, acc, cnt = _ce(logits, labels, ld)
    valid = labels >= 0
    nv = int(valid.sum())
    x = logits.double()
    lse = torch.logsumexp(x, 1)
    t = labels.clamp_min(0)
    ref_loss = lse - x.gather(1, t.view(-1, 1)).view(-1)
    ref_rank = PR.ranks(logits, t)
    ref_d = (torch.softmax(x, 1) - torch.nn.functional.one_hot(t, C).double()) / nv
    ref_d[~valid] = 0
    rl, rr, d = rl.cpu().double(), rr.cpu().long(), d.cpu().double()
    assert torch.equal(rr[valid], ref_rank[valid]) and bool((rr[~valid] == -1).all())
    # fp32 lse of O(10) logits: a few ulps of |lse|
    assert float((rl[valid] - ref_loss[valid]).abs().max()) <= 1e-5 * (1 + float(lse.abs().max()))
    assert bool((rl[~valid] == 0).all())
    # dlogits: bf16 rounding of a value with fp32 error ~1e-6 relative to 1 / B_valid
    assert float((d[:, :C] - ref_d).abs().max()) <= U * float(ref_d.abs().max()) + 1e-6 / nv
    assert bool((d[:, C:] == 0).all())
    mean = float(ref_loss[valid].mean())
    assert abs(float(loss) - mean) <= 1e-5 * abs(mean)
    h1, h5 = int((ref_rank[valid] < 1).sum()), int((ref_rank[valid] < 5).sum())
    assert cnt.tolist() == [1, nv, h1, h5]
    assert abs(float(acc) - float(loss)) == 0


def test_probe_ce_without_gradient_and_accumulation():
    logits = torch.randn(16, 1000, generator=torch.Generator().manual_seed(3))
    labels = torch.randint(0, 1000, (16,), generator=torch.Generator().manual_seed(4))
    _, rl, rr, loss, acc, cnt = _ce(logits, labels, 1000, grad=False)
    d, rl2, rr2, loss2, _, _ = _ce(logits, labels, 1000, grad=True)
    assert torch.equal(rl, rl2) and torch.equal(rr, rr2) and torch.equal(loss, loss2)


# ---- esvit_gemm_f32 against fp64 ---------------------------------------------------------------------------------
@pytest.mark.parametrize("M,N,K", [(128, 1000, 2304), (13, 16, 1920), (256, 1008, 3072), (40, 1000, 2048)])
def test_gemm_f32_matches_fp64(M, N, K):
    """|out - (a . b^T + bias)| <= (D 2^-23 + 2^-24) sum |a||b| + |bias| 2^-24 per element for bf16 operands (exact
    products, fp32 accumulation: DESIGN.md §4.4 / §4.20)"""
    from esvit_b200 import _lib
    from esvit_b200.ops import _p, _stream
    g = torch.Generator().manual_seed(M + N + K)
    a = torch.randn(M, K, generator=g).to(torch.bfloat16)
    b = (torch.randn(N, K, generator=g) * 0.05).to(torch.bfloat16)
    bias = torch.randn(N, generator=g)
    out = torch.empty(M, N, device="cuda")
    ad, bd, biasd = a.cuda(), b.cuda(), bias.cuda()
    _lib.call("esvit_gemm_f32", _p(ad), _p(bd), _p(biasd), _p(out), M, N, K, 0, _stream())
    ref = a.double() @ b.double().t() + bias.double()
    bound = (K * 2.0 ** -23 + 2.0 ** -24) * (a.double().abs() @ b.double().abs().t()) + bias.double().abs() * 2.0 ** -24
    err = (out.cpu().double() - ref).abs()
    assert bool((err <= bound).all()), float((err / bound).max())


def restart_from_checkpoint(ckp_path, run_variables=None, **kwargs):
    """utils.restart_from_checkpoint's loading sequence (utils.py:126-158): load_state_dict(strict=False), and
    without the keyword when the object does not take it"""
    checkpoint = torch.load(ckp_path, map_location="cpu", weights_only=False)
    for key, value in kwargs.items():
        try:
            value.load_state_dict(checkpoint[key], strict=False)
        except TypeError:
            value.load_state_dict(checkpoint[key])
    for var_name in run_variables or {}:
        if var_name in checkpoint:
            run_variables[var_name] = checkpoint[var_name]


# ---- LinearProbeStep against the reference trajectory -----------------------------------------------------------
def test_step_matches_reference_trajectory(G):
    """per step: loss within 4 x the largest bf16 logit bound; weight / bias / momentum updates within 8u of the
    update's norm (two bf16 operands per gradient product: u each; logit errors of 2u move the softmax by as much);
    validation hits equal the reference's exactly (the fixture keeps every outcome 4 x the bound away from a tie)"""
    from esvit_b200 import probe
    p = G["params"]
    clf, opt, step, losses, states = _run(G)
    x, y = G["train"]
    w, b, bw, bb = PR.init_classifier(p["D"], p["C"], p["init_seed"]) + (None, None)
    w0 = w
    lrs = PR.cosine_lrs(p["lr"], p["epochs"])
    nb = len(_batches(x, y, p["batch"]))
    for s, (xb, yb) in enumerate(_batches(x, y, p["batch"]) * p["epochs"]):
        delta = float(PR.logit_bound(w, xb).max())
        loss, w, b, bw, bb = PR.train_step(w, b, bw, bb, xb, yb, lrs[s // nb])
        ref = G["steps"][s]
        assert abs(loss - ref["loss"]) <= 1e-5 * abs(ref["loss"])  # the oracle is the reference's trajectory
        assert abs(float(losses[s]) - ref["loss"]) <= 4 * delta, (s, float(losses[s]), ref["loss"], delta)
        gw, gb, gbw, gbb = (t.cpu() for t in states[s])
        for name, o, r, r0 in (("weight", gw, w, w0), ("bias", gb, b, None), ("buf_w", gbw, bw, None),
                               ("buf_b", gbb, bb, None)):
            upd = (r - r0) if r0 is not None else r
            err = float((o.double() - r.double()).norm() / upd.double().norm())
            assert err <= 8 * U, (s, name, err)
    ev = probe.evaluate(_batches(*G["val"], p["batch"]), _Features(), clf, 4, False, [])
    for k in ("acc1", "acc5"):
        assert abs(ev[k] - G["validation"][k]) <= 1e-6 * G["validation"][k], (k, ev, G["validation"])


def test_evaluate_golden_weights_matches_reference(G):
    """validate_network on the reference's final weights: hits exactly, the loss within the bf16 logit bound"""
    from esvit_b200 import probe
    p = G["params"]
    x, y = G["train"]
    w, b, bw, bb = PR.init_classifier(p["D"], p["C"], p["init_seed"]) + (None, None)
    lrs = PR.cosine_lrs(p["lr"], p["epochs"])
    nb = len(_batches(x, y, p["batch"]))
    for s, (xb, yb) in enumerate(_batches(x, y, p["batch"]) * p["epochs"]):
        _, w, b, bw, bb = PR.train_step(w, b, bw, bb, xb, yb, lrs[s // nb])
    clf = probe.LinearClassifier(p["D"], p["C"]).cuda()
    clf.load_state_dict({"linear.weight": w, "linear.bias": b})
    xv, yv = G["val"]
    ev = probe.evaluate(_batches(xv, yv, p["batch"]), _Features(), clf, 4, False, [])
    ref = G["validation"]
    n = yv.numel()
    assert round(ev["acc1"] * n / 100) == round(ref["acc1"] * n / 100)
    assert round(ev["acc5"] * n / 100) == round(ref["acc5"] * n / 100)
    delta = float(PR.logit_bound(w, xv).max())
    assert abs(ev["loss"] - ref["loss"]) <= 2 * delta, (ev, ref, delta)
    # forward(): fp32 logits within the bound of the fp32 product
    lg = clf(xv.cuda()).cpu()
    assert lg.dtype == torch.float32 and lg.shape == (n, p["C"])
    assert bool(((lg - PR.forward(w, b, xv)).abs() <= PR.logit_bound(w, xv) + 1e-6).all())


def test_graph_replay_is_bit_identical_to_eager(G):
    """full batches (the ragged one dropped): three eager warm-up steps, then replays, against the eager step"""
    x, y = G["train"]
    B = G["params"]["batch"]
    xs, ys = x[:2 * B], y[:2 * B]
    runs = []
    for graph in (False, True, True):
        clf, opt, sched, step = _probe(G, graph)
        out = []
        for _ in range(3):
            for xb, yb in _batches(xs, ys, B):
                out.append(step(_as_images(xb), yb))
        torch.cuda.synchronize()
        runs.append((torch.stack(out), clf.linear.weight.detach().clone(), clf.linear.bias.detach().clone(),
                     opt.sweep.momentum_buffer[0].clone(), step.meter.counts.clone(), step.meter.acc.clone()))
        if graph:
            assert step._graph is not None
    for r in runs[1:]:
        for a, b in zip(runs[0], r):
            assert torch.equal(a, b)


def test_ragged_batch_runs_in_the_captured_graph(G):
    """the fixture's epochs in graph mode: the ragged batch of 37 replays the graph captured at 64 (padding rows
    labelled -1) and the trajectory stays on the eager one"""
    clf_e, _, _, le, se = _run(G, graph=False, epochs=3)
    clf_g, _, step, lg, sg = _run(G, graph=True, epochs=3)
    assert step._graph is not None and step._static[0].shape[0] == G["params"]["batch"]
    for s, (a, b) in enumerate(zip(se, sg)):
        for t, u in zip(a, b):
            assert float((t - u).abs().max()) <= 1e-5 * float(t.abs().max()) + 1e-7, s
        assert abs(float(le[s]) - float(lg[s])) <= 1e-5 * abs(float(le[s]))
    s = step.epoch_stats()
    assert s["images"] == 3 * G["params"]["n_train"] and s["batches"] == len(sg)


def test_checkpoint_round_trip_with_torch_sgd(G, tmp_path):
    """restart_from_checkpoint in both directions: a fused checkpoint resumes in torch.optim.SGD + CosineAnnealingLR
    and a torch checkpoint in ProbeSGD; both then continue training like an uninterrupted fused run"""
    p = G["params"]
    x, y = G["train"]
    bat = _batches(x, y, p["batch"])
    clf, opt, sched, step = _probe(G)
    for xb, yb in bat:
        step(_as_images(xb), yb)
    sched.step()
    ck = str(tmp_path / "fused.pth")
    torch.save({"epoch": 1, "state_dict": clf.state_dict(), "optimizer": opt.state_dict(),
                "scheduler": sched.state_dict()}, ck)
    # fused -> torch: the reference's loop continues one epoch
    lin = torch.nn.Linear(p["D"], p["C"]).cuda()
    tclf = torch.nn.Module()
    tclf.linear = lin
    topt = torch.optim.SGD(tclf.parameters(), 1.0, momentum=0.9, weight_decay=0)
    tsched = torch.optim.lr_scheduler.CosineAnnealingLR(topt, p["epochs"], eta_min=0)
    rv = {"epoch": 0}
    restart_from_checkpoint(ck, run_variables=rv, state_dict=tclf, optimizer=topt, scheduler=tsched)
    assert rv["epoch"] == 1 and topt.param_groups[0]["lr"] == opt.param_groups[0]["lr"]
    assert torch.equal(topt.state[lin.weight]["momentum_buffer"], opt.sweep.momentum_buffer[0])
    # torch -> fused
    ck2 = str(tmp_path / "torch.pth")
    torch.save({"epoch": 1, "state_dict": tclf.state_dict(), "optimizer": topt.state_dict(),
                "scheduler": tsched.state_dict()}, ck2)
    clf2, opt2, sched2, step2 = _probe(G, seed=123)
    restart_from_checkpoint(ck2, run_variables={"epoch": 0}, state_dict=clf2, optimizer=opt2, scheduler=sched2)
    assert opt2.param_groups[0]["lr"] == opt.param_groups[0]["lr"]
    assert sched2.last_epoch == sched.last_epoch
    # continue: uninterrupted fused, resumed fused (from torch) and resumed torch
    for xb, yb in bat:
        step(_as_images(xb), yb)
        step2(_as_images(xb), yb)
        topt.zero_grad()
        torch.nn.functional.cross_entropy(lin(xb.cuda()), yb.cuda()).backward()
        topt.step()
    torch.cuda.synchronize()
    assert torch.equal(clf.linear.weight, clf2.linear.weight) and torch.equal(clf.linear.bias, clf2.linear.bias)
    assert torch.equal(opt.sweep.momentum_buffer[0], opt2.sweep.momentum_buffer[0])
    w_f, w_t = clf.linear.weight.detach().double(), lin.weight.detach().double()
    upd = (w_f - w_t).norm() / w_f.norm()
    assert float(upd) <= 8 * U
    sd = opt.state_dict()
    assert list(sd["param_groups"][0]["params"]) == [0, 1] and sd["param_groups"][0]["weight_decay"] == 0
    assert set(sd["state"]) == {0, 1} and set(sd["state"][0]) == {"momentum_buffer"}


def test_swin_t_probe_features_inside_the_step():
    """Swin-T W7, n = 4 (D = 2304), on the backbone weights of the evaluation fixture's recipe at 224: the features the
    step feeds the classifier are bit-equal to a separate forward_return_n_last_blocks call"""
    from functools import partial
    from esvit_b200 import probe
    from esvit_b200.swin_transformer import SwinTransformer
    from oracle import golden as GD
    from oracle import swin as S
    spec = dict(S.SWIN_T_W7)
    m = SwinTransformer(img_size=224, num_classes=0, drop_path_rate=0.0,
                        norm_layer=partial(torch.nn.LayerNorm, eps=1e-6), **spec)
    m.load_state_dict(GD.seeded_state_dict(GD.recipe(m.state_dict()), 5))
    m = m.cuda().eval()
    depths = list(spec["depths"])
    torch.manual_seed(0)
    clf = probe.LinearClassifier(2304, 1000).cuda()
    opt = probe.ProbeSGD(clf.parameters(), 0.001)
    for graph in (False, True):
        step = probe.LinearProbeStep(m, clf, opt, 4, False, depths, use_cuda_graph=graph)
        for i in range(5 if graph else 1):
            x = torch.randn(8, 3, 224, 224, generator=torch.Generator().manual_seed(i)).cuda()
            loss = step(x, torch.randint(0, 1000, (8,), generator=torch.Generator().manual_seed(i)))
            with torch.no_grad():
                f = m.forward_return_n_last_blocks(x, 4, False, depths)
            torch.cuda.synchronize()
            assert torch.isfinite(loss) and torch.equal(step.last_features, f), (graph, i)


def test_invalid_input_raises_before_launch(G):
    from esvit_b200 import probe
    clf, opt, sched, step = _probe(G)
    x, y = G["train"]
    xb, yb = x[:16], y[:16]
    before = clf.linear.weight.detach().clone()
    with pytest.raises(ValueError):  # label >= num_labels
        step(_as_images(xb), torch.full((16,), G["params"]["C"]))
    with pytest.raises(ValueError):  # negative label
        step(_as_images(xb), yb - 100)
    with pytest.raises(ValueError):  # feature dimension differs from the classifier's
        step(_as_images(xb[:, :2296]), yb)
    with pytest.raises(ValueError):
        clf(xb[:, :2296].cuda())
    with pytest.raises(ValueError):  # label count differs from the batch
        step(_as_images(xb), yb[:15])
    with pytest.raises(ValueError):  # CUDA labels are not checked on the host
        step(_as_images(xb), yb.cuda())
    with pytest.raises(ValueError):
        probe.evaluate([(xb, yb + 2000)], _Features(), clf, 4, False, [])
    with pytest.raises(ValueError):  # weight decay
        probe.ProbeSGD(clf.parameters(), 0.1, weight_decay=1e-4)
    torch.cuda.synchronize()
    assert torch.equal(clf.linear.weight, before) and int(step.meter.counts[0]) == 0
