"""Host-side checks of set_train_forwards_in_flight: argument errors, delegation on the four module types, and the
choice of train plan instance (engine.Engine._train_instance) with plans built on the CPU and autograd nodes stood in
for by the tokens they keep (TrainPlan.claim); nothing is launched."""
import contextlib
import gc

import pytest
import torch

KW = dict(resolution=[160, 224], dim=16, in_dim=16, depths=[1, 1, 2, 1], num_heads=[1, 2, 4, 8], window_size=[7, 7, 5, 7])
DET_KW = dict(dim=16, in_dim=16, depths=[1, 1, 2, 1], num_heads=[1, 2, 4, 8])


def _models():
    from fastervit_b200 import detection, tracking
    from fastervit_b200.backbone import FasterViTBackbone
    from fastervit_b200.registry import create_model
    return {"classification": (m := create_model("faster_vit_0_any_res", **KW)), "classification.body": m,
            "backbone": (bb := FasterViTBackbone("faster_vit_0_any_res", out_indices=(1, 2), **KW)), "backbone.body": bb.body,
            "detection": (d := detection.build_fastervit("faster_vit_0_224", **DET_KW)), "detection.body": d,
            "tracking": (t := tracking.build_fastervit("faster_vit_0_224", tracking.FrozenBatchNorm2d, _LayerNorm2d,
                                                       **DET_KW)), "tracking.body": t}


class _LayerNorm2d(torch.nn.LayerNorm):   # timm's LayerNorm2d, as the tracking module classifies it
    pass


def test_arguments_and_delegation():
    from fastervit_b200.lib import FvitError
    ms = _models()
    for name in ("classification", "backbone", "detection", "tracking"):
        mod, body = ms[name], ms[name + ".body"]
        assert body._train_forwards_in_flight == 1
        assert mod.set_train_forwards_in_flight(3) is mod and body._train_forwards_in_flight == 3
        assert mod.set_train_forwards_in_flight() is mod and body._train_forwards_in_flight == 1
        for bad in (0, -2, 1.5, 2.0, "2", None, True):
            with pytest.raises(FvitError, match="set_train_forwards_in_flight"):
                mod.set_train_forwards_in_flight(bad)
        assert body._train_forwards_in_flight == 1
    import numpy as np
    assert ms["classification"].set_train_forwards_in_flight(np.int64(2))._train_forwards_in_flight == 2
    # deepcopy (ModelEmaV2) keeps the setting
    import copy
    assert copy.deepcopy(ms["detection"].set_train_forwards_in_flight(4))._train_forwards_in_flight == 4


@pytest.fixture
def engine_on_cpu(monkeypatch):
    """an Engine that builds real train plans on the CPU for a CUDA-looking input"""
    from fastervit_b200 import engine as E
    monkeypatch.setattr(E.Engine, "_check_weights", lambda self: ())
    monkeypatch.setattr(torch.cuda, "device", lambda dev: contextlib.nullcontext())

    def make(model, shape):
        class X:   # only its metadata is read
            is_cuda, dtype = True, torch.float32
            device = next(model.parameters()).device

            def dim(self):
                return 4
        X.shape = torch.Size(shape)
        return E.Engine(model), X()
    return make


def test_instance_choice_against_fake_nodes(engine_on_cpu):
    from fastervit_b200.registry import create_model
    m = create_model("faster_vit_0_any_res", **KW).train()
    eng, x = engine_on_cpu(m, (2, 3, 160, 224))
    m._engine = eng
    a = eng._plan(x)
    (key,) = eng.pools
    assert eng.plans[key] is a and eng.pools[key] == [a] and not a.in_flight()
    # n = 1: every forward gets the one instance, in flight or not (a second forward makes the first one stale)
    ta = a.claim()
    assert a.in_flight() and eng._plan(x) is a and len(eng.pools[key]) == 1
    a.release(ta)
    assert not a.in_flight()

    m.set_train_forwards_in_flight(2)
    ta = a.claim()
    with torch.no_grad():                  # (a forward moved the running means the first instance's pivots came from)
        for bn in (mod for mod in m.modules() if isinstance(mod, torch.nn.BatchNorm2d)):
            bn.running_mean.add_(0.25)
    b = eng._plan(x)                       # a is held: a second instance is built
    assert b is not a and eng.pools[key] == [a, b] and eng.plans[key] is a
    # every instance of a key centres its BatchNorm sums on the first one's pivots, so views round alike
    piv = [n for n in a.bufs.named if n.endswith(".pivot")]
    assert piv and all(torch.equal(a.bufs.named[n], b.bufs.named[n]) for n in piv)
    tb = b.claim()
    c = eng._plan(x)                       # both held, pool full: the oldest forward's instance
    assert c is a
    tc = c.claim()
    a.release(ta)                          # (the stale node's backward raises before it releases; a no-op anyway)
    assert a.in_flight()
    b.release(tb)                          # b's backward ran
    assert not b.in_flight() and eng._plan(x) is b
    del tc
    gc.collect()
    assert not a.in_flight() and eng._plan(x) is a   # a node freed without a backward frees its instance
    assert len(eng.pools[key]) == 2

    # three forwards, the first one's outputs dropped before the third: two instances, not three
    m.set_train_forwards_in_flight(3)
    t1 = eng._plan(x).claim()
    p2 = eng._plan(x)
    t2 = p2.claim()
    del t1
    p3 = eng._plan(x)
    assert p3 is a and len(eng.pools[key]) == 2
    t3 = p3.claim()
    assert eng._plan(x) not in (a, p2) and len(eng.pools[key]) == 3     # (now all three held)
    # a steady loop of two forwards then their backwards reuses the instances
    del t2, t3
    pool = list(eng.pools[key])
    for _ in range(3):
        p, q = eng._plan(x), None
        tp = p.claim()
        q = eng._plan(x)
        tq = q.claim()
        assert p is not q and p in pool and q in pool
        p.release(tp)
        q.release(tq)
    assert eng.pools[key] == pool
    # lowering the bound drops the last instances; the key's first one stays the plan the cache lists
    m.set_train_forwards_in_flight(1)
    assert eng.pools[key] == [a] and eng.plans[key] is a


def test_eval_grad_plans_are_not_pooled_and_lru_drops_a_keys_instances(engine_on_cpu):
    from fastervit_b200 import detection
    from fastervit_b200.registry import create_model
    m = create_model("faster_vit_0_any_res", **KW).eval()
    eng, x = engine_on_cpu(m, (2, 3, 160, 224))
    assert eng.eval_grad_plan(x) is eng.eval_grad_plan(x) and not eng.pools

    det = detection.build_fastervit("faster_vit_0_224", **DET_KW).train().set_train_forwards_in_flight(2)
    eng, x1 = engine_on_cpu(det, (1, 3, 96, 160))
    _, x2 = engine_on_cpu(det, (1, 3, 64, 96))
    det._engine = eng
    spec = dict(kind="levels", outs=tuple((i, det._level_norm(i)) for i in det.out_indices), frozen=-1)
    p1 = eng._plan(x1, spec)
    t1 = p1.claim()
    q1 = eng._plan(x1, spec)
    assert q1 is not p1 and len(eng.pools) == 1
    eng._plan(x2, spec)
    assert len(eng.plans) == len(eng.pools) == 2
    det.set_plan_cache_size(1)             # the first shape's key goes, both its instances with it
    assert len(eng.plans) == len(eng.pools) == 1 and all(k[0] == (1, 3, 64, 96) for k in eng.pools)
    assert p1.in_flight()                  # (its node keeps it until its backward)
    del t1
