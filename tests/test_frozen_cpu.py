"""Frozen parameters (requires_grad=False) on the host side: the float64 optimiser step against torch's AdamW / Adam and
clip_grad_norm_ with grad=None parameters, the frozen set and AdamW ranges, the backward plan's truncation, the
gradient buckets over gloo world 2, and the optimizer checkpoint against the reference's get_optimizer."""
import os
import socket
import types

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import optim_reference as OR
from oracle import ref_harness
from open_musiclm_b200.dist_utils import BucketReducer, drop_frozen_buckets, plan_buckets
from open_musiclm_b200.trainer import HotPathTrainer, frozen_parameter_names, live_ranges
from test_dist_cpu import _toy_layout


# ------------------------------------------------------------------------------------------------ optimiser step
def _arena(shapes):
    """Flat layout of `shapes` as the engine orders it: 64-aligned, ndim >= 2 first (decayed: [0, n_decay))."""
    offs, off = {}, 0
    for i in sorted(range(len(shapes)), key=lambda i: len(shapes[i]) < 2):
        if len(shapes[i]) < 2 and "n_decay" not in locals():
            n_decay = off
        offs[i] = off
        off = (off + torch.Size(shapes[i]).numel() + 63) // 64 * 64
    return offs, off, n_decay


@pytest.mark.parametrize("wd", [0.0, 0.01])
@pytest.mark.parametrize("max_norm", [0.05, 1e6])
def test_float64_step_with_frozen_members_matches_torch(wd, max_norm):
    """Six steps of OR.adamw_update over an arena whose frozen ranges have zero gradient equal torch's optimizer (the
    reference's get_optimizer layout) and clip_grad_norm_ over parameters whose frozen members keep grad None."""
    shapes = [(7, 5), (3, 70), (11,), (4, 4, 3), (9,), (65,)]
    frozen = {1, 4}
    offs, total, n_decay = _arena(shapes)
    gen = torch.Generator().manual_seed(3)
    params = [torch.nn.Parameter(torch.randn(s, generator=gen, dtype=torch.float64)) for s in shapes]
    opt = OR.reference_optimizer(params, lr=1e-2, wd=wd)
    p = torch.zeros(total, dtype=torch.float64)
    for i, q in enumerate(params):
        p[offs[i]:offs[i] + q.numel()] = q.detach().reshape(-1)
    m, v = torch.zeros_like(p), torch.zeros_like(p)
    spans = [(offs[i], offs[i] + params[i].numel()) for i in frozen]
    for step in range(6):
        g = torch.zeros(total, dtype=torch.float64)
        for i, q in enumerate(params):
            if i in frozen:
                q.grad = None
            else:
                q.grad = torch.randn(q.shape, generator=gen, dtype=torch.float64) * (10.0 ** (i - 3))
                g[offs[i]:offs[i] + q.numel()] = q.grad.reshape(-1)
        norm_t = float(torch.nn.utils.clip_grad_norm_(params, max_norm))
        opt.step()
        p, m, v, norm = OR.adamw_update(p, g, m, v, t=step + 1, lr=1e-2, wd=wd, n_decay=n_decay, max_grad_norm=max_norm, frozen=spans)
        assert abs(norm - norm_t) <= 1e-12 * norm_t
        for i, q in enumerate(params):
            got = p[offs[i]:offs[i] + q.numel()].view(q.shape)
            assert torch.allclose(got, q.detach(), rtol=1e-12, atol=1e-15), (step, i)
            if i in frozen:
                assert q not in opt.state
                assert not bool(m[offs[i]:offs[i] + q.numel()].any()) and not bool(v[offs[i]:offs[i] + q.numel()].any())
            else:
                st = opt.state[q]
                assert torch.allclose(m[offs[i]:offs[i] + q.numel()].view(q.shape), st["exp_avg"], rtol=1e-12, atol=1e-18)
                assert torch.allclose(v[offs[i]:offs[i] + q.numel()].view(q.shape), st["exp_avg_sq"], rtol=1e-12, atol=1e-24)


# ------------------------------------------------------------------------------------------------ frozen set
def test_frozen_names_follow_requires_grad():
    names = ["logit_weights.0", "logit_weights.1", "embeddings.0.weight", "start_tokens.0", "transformer.norm.gamma"]
    rg = {n: True for n in names}
    assert frozen_parameter_names(names, [0.0, 1.0], rg) == {"logit_weights.0"}
    rg["embeddings.0.weight"] = rg["start_tokens.0"] = rg["logit_weights.1"] = False
    assert frozen_parameter_names(names, [0.0, 1.0], rg) == {"logit_weights.0", "logit_weights.1", "embeddings.0.weight", "start_tokens.0"}
    assert frozen_parameter_names(names, [1.0, 1.0]) == set()
    layout = {n: 100 * i for i, n in enumerate(names)}
    spans = [(layout[n], layout[n] + 64) for n in frozen_parameter_names(names, [0.0, 1.0], rg)]
    assert live_ranges(500, spans) == [(64, 100), (164, 200), (264, 300), (364, 500)]


def test_trainer_reads_requires_grad_once():
    """train_step refuses to run after a requires_grad flag changed (checked before any device work)."""
    m = torch.nn.Linear(3, 2)
    fake = types.SimpleNamespace(transformer=m, grad_accum_every=1, eng=None,
                                 _requires_grad={n: p.requires_grad for n, p in m.named_parameters()})
    m.bias.requires_grad_(False)
    with pytest.raises(RuntimeError, match="requires_grad changed"):
        HotPathTrainer.train_step(fake, [[]])


# ------------------------------------------------------------------------------------------------ backward plan
def _plan(frozen, depth=4, bias="continuous", conv=True):
    from open_musiclm_b200.engine import _BackwardPlan
    names = ["embeddings.0.weight", "start_tokens.0", "logit_weights.0", "transformer.norm.gamma"]
    ff = ["2.0.gamma", "2.1.weight", "2.2.ds_conv.weight", "2.4.gamma", "2.6.weight"] if conv else \
         ["2.0.gamma", "2.1.weight", "2.3.gamma", "2.5.weight"]
    for l in range(depth):
        names += [f"transformer.layers.{l}.{k}" for k in ["0.norm.gamma", "0.to_q.weight", "0.to_kv.weight", "0.q_scale", "0.k_scale",
                                                          "0.to_out.0.weight"] + ff]
    if bias == "continuous":
        names += [f"transformer.rel_pos_bias.net.{j}.0.{k}" for j in range(3) for k in ("weight", "bias")] + \
                 ["transformer.rel_pos_bias.net.3.weight", "transformer.rel_pos_bias.net.3.bias"]
    elif bias == "t5":
        names += ["transformer.rel_pos_bias.relative_attention_bias.weight"]
    eng = types.SimpleNamespace(layout={n: i for i, n in enumerate(names)}, L=depth)
    eng.ffk = (dict(g1="2.0.gamma", w1="2.1.weight", conv="2.2.ds_conv.weight", gin="2.4.gamma", w2="2.6.weight") if conv
               else dict(g1="2.0.gamma", w1="2.1.weight", conv=None, gin="2.3.gamma", w2="2.5.weight"))
    fz = {n for n in names if any(n.startswith(f) for f in frozen)} if frozen != "all" else set(names)
    return _BackwardPlan(eng, fz), names


def test_backward_plan_truncates_below_the_lowest_trainable_layer():
    rows = ("embeddings.", "start_tokens.")
    bp, _ = _plan(rows + ("transformer.rel_pos_bias.",) + tuple(f"transformer.layers.{l}." for l in range(3)))
    assert bp.run == [False, False, False, True] and not bp.dtable and not bp.rows and bp.final_norm
    assert not bp.steps[3]["g_in"] and bp.steps[3]["ln_a"] and bp.steps[3]["attn"]      # (ln_a: layer 3's own gamma)
    # the bias MLP trains: every layer's dS is needed, but no gradient has to reach the layers' inputs below layer 1
    bp, _ = _plan(rows + tuple(f"transformer.layers.{l}." for l in range(4)))
    assert bp.run == [True] * 4 and bp.dtable and [s["g_in"] for s in bp.steps] == [False, True, True, True]
    assert bp.steps[0]["attn"] and not bp.steps[0]["qk"]
    # only the feed-forward output matrix of layer 2: layers 0, 1 are skipped, layer 2 runs no attention backward
    bp, names = _plan(rows + ("transformer.rel_pos_bias.", "transformer.layers.0.", "transformer.layers.1.", "transformer.layers.3.",
                              "transformer.norm.", "logit_weights.") + tuple(f"transformer.layers.2.{k}" for k in
                                                                             ("0.", "2.0.", "2.1.", "2.2.", "2.4.")))
    assert bp.run == [False, False, True, True] and bp.final_norm
    assert not bp.steps[2]["ffn"] and not bp.steps[2]["attn"] and not bp.steps[2]["ln_f"]
    assert bp.steps[3]["g_in"] and bp.steps[3]["ln_a"]
    # 'none' has no table parameters; T5 trains its table only through its one parameter
    bp, _ = _plan(rows, bias="none")
    assert not bp.dtable
    bp, _ = _plan(rows, bias="t5")
    assert bp.dtable
    bp, _ = _plan(rows + ("transformer.rel_pos_bias.",), bias="t5", conv=False)
    assert not bp.dtable
    # a partly frozen set of row tables; everything frozen runs nothing
    bp, _ = _plan(("embeddings.",))
    assert bp.rows and bp.rows_partial and bp.run == [True] * 4
    bp, _ = _plan("all")
    assert not any(bp.run) and not bp.final_norm and not bp.rows and not bp.dtable


# ------------------------------------------------------------------------------------------------ gradient buckets
def _frozen_bucket_worker(rank, world, port, out):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    layout, sizes, total = _toy_layout(4)
    frozen = {n for n in layout if n.startswith(("logit_weights.", "transformer.layers.0.", "transformer.layers.1."))
              and n.endswith("weight") or n.startswith("logit_weights.")}
    plan = plan_buckets(layout, sizes, total, 4, min_elems=500)
    live = drop_frozen_buckets(plan, [(layout[n], layout[n] + sizes[n]) for n in layout if n not in frozen])
    g = torch.Generator().manual_seed(100 + rank)
    flat = torch.randn(total, generator=g)
    calls = []
    red = BucketReducer(flat, live, None, side_stream=None)
    orig = red._reduce
    red._reduce = lambda view: (calls.append(view.numel()), orig(view))
    red.begin()
    red.fire("heads")
    for l in reversed(range(4)):
        red.fire(f"layer{l}")
    red.fire("tail")
    red.join()
    if rank == 0:
        torch.save(dict(flat=flat, plan=plan, live=live, calls=calls), out)
    dist.destroy_process_group()


def test_frozen_buckets_are_not_communicated(tmp_path):
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    out = str(tmp_path / "flat.pt")
    mp.spawn(_frozen_bucket_worker, args=(2, port, out), nprocs=2, join=True)
    r = torch.load(out)
    _, _, total = _toy_layout(4)
    mine = torch.randn(total, generator=torch.Generator().manual_seed(100))
    both = mine + torch.randn(total, generator=torch.Generator().manual_seed(101))
    dropped = [t for t, _ in r["plan"] if t not in dict(r["live"])]
    assert "heads" in dropped and "layer0" in dropped and "tail" not in dropped
    assert sum(r["calls"]) == sum(hi - lo for _, sl in r["live"] for lo, hi in sl)
    for t, sl in r["plan"]:
        for lo, hi in sl:
            want = mine if t in dropped else both
            assert torch.equal(r["flat"][lo:hi], want[lo:hi]), t


# ------------------------------------------------------------------------------------------------ checkpoint
@pytest.mark.parametrize("wd", [0.0, 0.01])
def test_checkpoint_with_frozen_parameters_loads_into_get_optimizer(tmp_path, wd):
    """save() of a trainer with frozen parameters writes the reference's optimizer file with no state for them; it loads
    into get_optimizer(transformer.parameters()) (or the same torch optimizer when no reference checkout is present),
    and HotPathTrainer.load() reads it back."""
    torch.manual_seed(0)
    model = torch.nn.Sequential(torch.nn.Linear(6, 5), torch.nn.LayerNorm(5), torch.nn.Linear(5, 3))
    names = [n for n, _ in model.named_parameters()]
    frozen = {"0.weight", "1.bias"}
    for n, p in model.named_parameters():
        p.requires_grad_(n not in frozen)
    offs, off = {}, 0
    for n, p in model.named_parameters():
        offs[n] = off
        off += (p.numel() + 63) // 64 * 64
    gen = torch.Generator().manual_seed(1)
    eng = types.SimpleNamespace(layout=offs, adam_m=torch.randn(off, generator=gen).abs(), adam_v=torch.randn(off, generator=gen).abs(),
                                arena_g=torch.zeros(off), refresh_packed=lambda force=False: None, dev=torch.device("cpu"))
    fake = types.SimpleNamespace(transformer=model, eng=eng, frozen=frozen, steps=3, lr=1e-3, wd=wd, betas=(0.9, 0.99), eps=1e-8,
                                 lr_warmup=0)
    fake._gather_optimizer_state = lambda: None
    fake._torch_optimizer = lambda: HotPathTrainer._torch_optimizer(fake)
    fake._lr_factor = lambda s: HotPathTrainer._lr_factor(fake, s)
    paths = [str(tmp_path / f) for f in ("model.pt", "optim.pt")]
    HotPathTrainer.save(fake, *paths)
    params = list(model.parameters())
    if ref_harness.available():
        ref_harness.import_reference()
        from open_musiclm import optimizer as ref_opt
        opt = ref_opt.get_optimizer(params, lr=1e-3, wd=wd)
    else:
        opt = OR.reference_optimizer(params, lr=1e-3, wd=wd)
    opt.load_state_dict(torch.load(paths[1]))
    for n, p in model.named_parameters():
        assert (p in opt.state) == (n not in frozen), n
        if n not in frozen:
            o = offs[n]
            assert torch.equal(opt.state[p]["exp_avg"], eng.adam_m[o:o + p.numel()].view(p.shape))
            assert torch.equal(opt.state[p]["exp_avg_sq"], eng.adam_v[o:o + p.numel()].view(p.shape))
    m0, v0 = eng.adam_m.clone(), eng.adam_v.clone()
    assert HotPathTrainer.load(fake, *paths) == 3
    for n, p in model.named_parameters():
        o, k = offs[n], p.numel()
        if n in frozen:
            assert not bool(eng.adam_m[o:o + k].any()) and not bool(eng.adam_v[o:o + k].any())
        else:
            assert torch.equal(eng.adam_m[o:o + k], m0[o:o + k]) and torch.equal(eng.adam_v[o:o + k], v0[o:o + k])
