"""Generate tests/golden/esvit_probe.pt by RUNNING THE UNMODIFIED REFERENCE's linear-probe code.

TEST INFRASTRUCTURE.  Usage (ESVIT_REFERENCE = a reference checkout, else oracle/_ref/):

    python -m oracle.make_golden_probe

eval_linear.py's LinearClassifier, train() and validate_network() with utils.accuracy / MetricLogger (AST-extracted,
oracle/probe.py) on the CPU in fp32, with torch.optim.SGD(momentum 0.9, weight_decay 0) and CosineAnnealingLR(epochs,
eta_min=0) stepped per epoch as the script's main loop does.  The frozen backbone is the identity on seeded synthetic
features (D = 2304, the Swin-T n = 4 width; C = 1000, 24 classes used): the loader yields the features themselves.
Two epochs of three steps, batch 64 with a ragged last batch of 37; every step's loss, bias, momentum buffers and a
seeded sample of the weight (oracle.golden.sample), the per-epoch lr and the validation dict are stored.  The validation
rows are the first 150 of a seeded pool whose top-1 / top-5 outcome under the trained weights no logits within 4x the
bf16 bound (oracle.probe.logit_bound) could change: hit counts then compare exactly.  oracle/probe.py is asserted
against every stored value while the file is written.
"""
from __future__ import annotations

import os
import sys

import torch

from . import golden as GD
from . import probe as PR
from . import reference_import as R
from .eval import cpu_cuda_shim

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "esvit_probe.pt")

D, C, USED = 2304, 1000, 24
CENTRE_SEED, INIT_SEED, TRAIN_SEED, VAL_SEED = 10, 11, 12, 13
BATCH, N_TRAIN, N_VAL, N_POOL = 64, 2 * 64 + 37, 150, 3000
EPOCHS, LR = 2, 0.003
MARGIN = 4.0


class _Identity:
    """the frozen backbone: the loader already yields the probe features"""

    def forward_return_n_last_blocks(self, x, n, avgpool, depths):
        return x


def _batches(x, y):
    return [(x[r:r + BATCH], y[r:r + BATCH]) for r in range(0, x.shape[0], BATCH)]


class _Recorder(torch.optim.SGD):
    """torch.optim.SGD that records the state after every step"""

    def __init__(self, *a, log=None, **kw):
        super().__init__(*a, **kw)
        self.log = log

    def step(self, closure=None):
        out = super().step(closure)
        w, b = self.param_groups[0]["params"]
        self.log.append(dict(weight=w.detach().clone(), bias=b.detach().clone(),
                             buf_w=self.state[w]["momentum_buffer"].clone(),
                             buf_b=self.state[b]["momentum_buffer"].clone()))
        return out


def generate():
    ref = PR.reference_probe()
    xtr, ytr = PR.probe_features(CENTRE_SEED, TRAIN_SEED, N_TRAIN, D, USED)
    torch.manual_seed(INIT_SEED)
    clf = ref["LinearClassifier"](D, C)
    w0, b0 = PR.init_classifier(D, C, INIT_SEED)
    assert torch.equal(clf.linear.weight, w0) and torch.equal(clf.linear.bias, b0)
    log = []
    opt = _Recorder(clf.parameters(), LR, momentum=0.9, weight_decay=0, log=log)
    sched = torch.optim.lr_scheduler.CosineAnnealingLR(opt, EPOCHS, eta_min=0)
    lrs, train_stats, losses = [], [], []
    model = _Identity()
    def record(module, args, out):  # the loss of each train() step (nn.CrossEntropyLoss()(output, target))
        if isinstance(module, torch.nn.CrossEntropyLoss) and recording:
            losses.append(float(out.detach()))

    recording = True
    hook = torch.nn.modules.module.register_module_forward_hook(record)
    saved_sync = torch.cuda.synchronize
    torch.cuda.synchronize = lambda *a, **k: None
    try:
        with cpu_cuda_shim():
            for epoch in range(EPOCHS):
                lrs.append(opt.param_groups[0]["lr"])
                train_stats.append(ref["train"](model, clf, opt, _batches(xtr, ytr), epoch, 4, False, []))
                sched.step()
            recording = False
            # the validation rows: the first N_VAL of a seeded pool whose top-1 / top-5 outcomes under the trained
            # weights no logits within MARGIN x the bf16 bound (oracle.probe.logit_bound) could change
            wf, bf = clf.linear.weight.detach().clone(), clf.linear.bias.detach().clone()
            xpo, ypo = PR.probe_features(CENTRE_SEED, VAL_SEED, N_POOL, D, USED)
            ok = PR.decided(PR.forward(wf, bf, xpo), ypo, MARGIN * PR.logit_bound(wf, xpo))
            keep = ok.nonzero().view(-1)[:N_VAL]
            assert keep.numel() == N_VAL, int(ok.sum())
            xva, yva = xpo[keep], ypo[keep]
            val = ref["validate_network"](_batches(xva, yva), model, clf, 4, False, [])
    finally:
        torch.cuda.synchronize = saved_sync
        hook.remove()
    steps_per_epoch = len(_batches(xtr, ytr))
    assert len(log) == EPOCHS * steps_per_epoch and len(losses) == len(log)
    assert lrs == PR.cosine_lrs(LR, EPOCHS), (lrs, PR.cosine_lrs(LR, EPOCHS))

    # the oracle reproduces the trajectory
    w, b, bw, bb = w0, b0, None, None
    for s, (x, y) in enumerate(_batches(xtr, ytr) * EPOCHS):
        loss, w, b, bw, bb = PR.train_step(w, b, bw, bb, x, y, lrs[s // steps_per_epoch])
        assert abs(loss - losses[s]) <= 1e-5 * abs(losses[s]), (s, loss, losses[s])
        for name, o in (("weight", w), ("bias", b), ("buf_w", bw), ("buf_b", bb)):
            r = log[s][name]
            assert torch.allclose(o, r, rtol=1e-4, atol=2e-6), (s, name, float((o - r).abs().max()))
    assert torch.equal(wf, log[-1]["weight"]) and torch.equal(bf, log[-1]["bias"])
    ov = PR.validate(wf, bf, xva, yva, BATCH)
    for k in ("loss", "acc1", "acc5"):  # MetricLogger sums the per-batch percentages in float
        assert abs(ov[k] - val[k]) <= 1e-6 * abs(val[k]), (k, ov, val)

    steps = [dict(loss=losses[s], bias=log[s]["bias"], buf_b=log[s]["buf_b"],
                  weight=GD.sample(log[s]["weight"], seed=s), buf_w=GD.sample(log[s]["buf_w"], seed=100 + s),
                  weight_norm=float(log[s]["weight"].double().norm()), buf_w_norm=float(log[s]["buf_w"].double().norm()))
             for s in range(len(log))]
    return dict(params=dict(D=D, C=C, classes_used=USED, centre_seed=CENTRE_SEED, init_seed=INIT_SEED,
                            train_seed=TRAIN_SEED, val_seed=VAL_SEED, batch=BATCH, n_train=N_TRAIN, n_pool=N_POOL,
                            epochs=EPOCHS, lr=LR, margin=MARGIN),
                val_rows=keep.to(torch.int16),
                lrs=lrs, steps=steps, train_stats=train_stats, validation=val,
                final=dict(weight=GD.sample(wf, seed=999), bias=bf.clone()),
                generator="oracle/make_golden_probe.py (reference run on CPU fp32, torch %s)" % torch.__version__)


def load(path: str) -> dict:
    """the fixture with its features rebuilt from their seeds"""
    G = torch.load(path, map_location="cpu", weights_only=False)
    p = G["params"]
    G["train"] = PR.probe_features(p["centre_seed"], p["train_seed"], p["n_train"], p["D"], p["classes_used"])
    x, y = PR.probe_features(p["centre_seed"], p["val_seed"], p["n_pool"], p["D"], p["classes_used"])
    rows = G["val_rows"].long()
    G["val"] = (x[rows], y[rows])
    return G


if __name__ == "__main__":
    if not R.available():
        sys.exit("reference tree not found: set ESVIT_REFERENCE to a checkout of microsoft/esvit")
    out = generate()
    torch.save(out, OUT)
    print("wrote", OUT, os.path.getsize(OUT) // 1024, "KiB; validation", out["validation"])
