"""Conversion over several ranks (``convert.convert_utterances`` / ``convert_slices`` with ``group=``, ``shard.plan_batches``,
``shard.gather_ragged``, ``shard.run_sharded``, ``shard.check_generator``).

CPU: the planner's properties, a 3-rank gloo round trip of the ragged gather with uneven sizes and an idle rank, a failing rank
that makes every rank raise, mismatched generators, and argument errors raised on every rank before any collective.  GPU: two
ranks (NCCL on two GPUs, else gloo with both ranks on cuda:0) convert the six slices of ``tests/test_convert.py`` with its small
chain, against the single-process call.  Child processes are joined with timeouts and terminated if they outlive them."""
import math
import os
import socket
from datetime import timedelta

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from ns2vc_b200 import api, convert, shard

SR = 44100
STEPS = 4


def _plans(n, seed):
    g = np.random.default_rng(seed)
    plans = [convert.frame_plan(int(g.integers(8000, 200000)), SR) for _ in range(n)]
    return plans, [int(x) for x in g.integers(20, 400, n)]


def _cost(b, plans, sl):
    return len(b) * shard.sample_step_flops(max(plans[i]["T"] for i in b), max(sl[i] for i in b))


# ------------------------------------------------------------------------------------------------------------- planner (CPU)
@pytest.mark.parametrize("n,world,max_batch", [(64, 8, 8), (64, 2, 8), (37, 3, 8), (16, 4, 3), (5, 2, 8), (9, 4, 1), (3, 8, 8),
                                               (1, 2, 8)])
def test_plan_covers_each_utterance_once_and_balances(n, world, max_batch):
    plans, sl = _plans(n, n * 31 + world)
    plan = shard.plan_batches(plans, sl, world, max_batch)
    assert len(plan) == world
    flat = [i for batches in plan for b in batches for i in b]
    assert sorted(flat) == list(range(n)), "every index exactly once"
    assert plan == shard.plan_batches(plans, sl, world, max_batch), "deterministic"
    cap = min(max_batch, math.ceil(n / world))
    assert all(1 <= len(b) <= cap for batches in plan for b in batches)
    loads = [sum(_cost(b, plans, sl) for b in batches) for batches in plan]
    worst = max(_cost(b, plans, sl) for batches in plan for b in batches)
    assert max(loads) <= min(loads) + worst, f"loads {loads}, costliest batch {worst}"
    if n < world:
        assert sum(1 for batches in plan if not batches) == world - n and all(len(batches) <= 1 for batches in plan)
    elif n >= world * cap:
        assert all(plan), "every rank has work"


def test_plan_of_one_rank_is_batch_plan():
    for n, max_batch in ((64, 8), (7, 3), (1, 8), (10, 100)):
        plans, sl = _plans(n, n)
        assert shard.plan_batches(plans, sl, 1, max_batch) == [api.batch_plan([p["n24"] for p in plans], max_batch)]


def test_plan_assigns_costliest_batch_first_to_least_loaded_rank():
    plans = [dict(n24=t * 256, T=t, n16=0, units=0) for t in (1000, 900, 400, 300, 200, 100)]
    sl = [100] * 6
    plan = shard.plan_batches(plans, sl, 2, 2)      # batches [0, 1], [2, 3], [4, 5]; the first outweighs the other two together
    assert plan == [[[0, 1]], [[2, 3], [4, 5]]]
    assert shard.plan_batches(plans, sl, 3, 8) == [[[0, 1]], [[2, 3]], [[4, 5]]]
    with pytest.raises(ValueError):
        shard.plan_batches(plans, sl, 0, 2)
    with pytest.raises(ValueError):
        shard.plan_batches(plans, sl, 2, 0)
    with pytest.raises(ValueError):
        shard.plan_batches(plans, sl[:5], 2, 2)


# ---------------------------------------------------------------------------------------------------------- process harness
def _entry(target, rank, world, port, backend, q, args):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    kw = {}
    if backend == "nccl":
        kw["device_id"] = torch.device("cuda", rank)
        torch.cuda.set_device(rank)
    elif torch.cuda.is_available():
        torch.cuda.set_device(0)
    dist.init_process_group(backend, rank=rank, world_size=world, timeout=timedelta(seconds=90), **kw)
    try:
        q.put((rank, target(rank, world, *args)))
    except BaseException as e:
        q.put((rank, f"worker raised {type(e).__name__}: {e}"))
    finally:
        dist.destroy_process_group()


def _run(target, world, *args, backend="gloo", timeout=180):
    """Runs ``target(rank, world, *args)`` in ``world`` spawned processes of one process group; returns the results by rank."""
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_entry, args=(target, r, world, port, backend, q, args)) for r in range(world)]
    for p in procs:
        p.start()
    try:
        res = dict(q.get(timeout=timeout) for _ in procs)
    finally:
        for p in procs:
            p.join(timeout=60)
            if p.is_alive():
                p.terminate()
                p.join(timeout=10)
    assert all(p.exitcode == 0 for p in procs), [p.exitcode for p in procs]
    return [res[r] for r in range(world)]


# ----------------------------------------------------------------------------------------------------- collectives (CPU, gloo)
def _value(i, shape):
    return torch.arange(math.prod(shape), dtype=torch.float32).view(shape) * 0.5 + 1000 * i + 1


SHAPES = [(7,), (3, 5), (1,), (40,), (2, 2), (13,), (6,)]
PLAN = [[[3, 0], [5]], [], [[1, 4], [6], [2]]]          # rank 1 idle; packed sizes 61, 0, 27


def _gather_worker(rank, world):
    local = [_value(i, SHAPES[i]) for b in PLAN[rank] for i in b]
    got = shard.gather_ragged(local, PLAN, SHAPES, dist.group.WORLD)
    ok = len(got) == len(SHAPES) and all(torch.equal(g, _value(i, s)) for i, (g, s) in enumerate(zip(got, SHAPES)))
    # a plan from the planner with fewer utterances than ranks, 1-D sizes
    plans, sl = _plans(2, 4)
    plan = shard.plan_batches(plans, sl, world, 8)
    sizes = [p["T"] for p in plans]
    got2 = shard.run_sharded(lambda idx: [_value(i, (sizes[i],)) for i in idx], plan, sizes, dist.group.WORLD)
    ok2 = sum(1 for b in plan if not b) == 1 and all(torch.equal(g, _value(i, (s,))) for i, (g, s) in enumerate(zip(got2, sizes)))
    return ok, ok2


def test_gather_ragged_three_ranks_uneven_sizes_and_an_idle_rank():
    assert _run(_gather_worker, 3) == [(True, True)] * 3


def _failing_worker(rank, world):
    plans, sl = _plans(9, 1)
    plan = shard.plan_batches(plans, sl, world, 8)

    def work(idx):
        if rank == 1:
            raise AssertionError("sampler produced NaN")
        return [torch.zeros(plans[i]["T"]) for i in idx]
    try:
        shard.run_sharded(work, plan, [p["T"] for p in plans], dist.group.WORLD)
    except RuntimeError as e:
        return str(e)
    return "no error"


def test_a_failing_rank_makes_every_rank_raise():
    msgs = _run(_failing_worker, 3)
    for r, m in enumerate(msgs):
        assert m.startswith("sharded run failed on rank(s) [1]"), f"rank {r}: {m}"
    assert "AssertionError: sampler produced NaN" in msgs[1]


def _generator_worker(rank, world):
    shard.check_generator(torch.Generator().manual_seed(7), dist.group.WORLD)          # equal seeds pass
    out = []
    try:
        shard.check_generator(torch.Generator().manual_seed(7 + (rank == 2)), dist.group.WORLD)
        out.append("no error")
    except ValueError as e:
        out.append(str(e))
    mel = torch.zeros(100, 30)
    for wavs, kw in (([torch.zeros(300)], {}), ([torch.zeros(20000)], dict(method="ddim")), ([], {})):
        try:
            convert.convert_utterances(None, None, None, None, wavs, SR, mel, group=dist.group.WORLD, **kw)
            out.append("no error")
        except ValueError as e:
            out.append(type(e).__name__)
    return out


def test_mismatched_generators_and_bad_arguments_raise_on_every_rank():
    for r, out in enumerate(_run(_generator_worker, 3)):
        assert "call torch.manual_seed with the same seed on every rank" in out[0], f"rank {r}: {out[0]}"
        assert out[1:] == ["ValueError"] * 3, f"rank {r}: {out}"


# --------------------------------------------------------------------------------------------------------------------- GPU
def _chain(dev):
    """The small chain and the six slices of tests/test_convert.py, with the models on ``dev``."""
    from test_convert import DURATIONS, PRE_CFG
    from ns2vc_b200.arch import UNetConfig
    from ns2vc_b200.content import ContentVec
    from ns2vc_b200.pre_model import Pre_model
    from ns2vc_b200.synth import CONTENTVEC_SMALL, make_contentvec_state_dict, make_pre_state_dict, make_state_dict, make_vocos_state_dict
    from ns2vc_b200.unet import UNet1DConditionModel
    from ns2vc_b200.vocoder import Vocos
    cv = ContentVec.from_state_dict(make_contentvec_state_dict(0, "trained_like", **CONTENTVEC_SMALL),
                                    num_heads=CONTENTVEC_SMALL["num_heads"]).to(dev)
    pre = Pre_model(PRE_CFG)
    pre.load_state_dict(make_pre_state_dict(PRE_CFG, 0))
    pre = pre.to(dev).eval()
    c = UNetConfig(in_channels=132, out_channels=100, block_out_channels=(32, 64, 64, 96), norm_num_groups=8, cross_attention_dim=32,
                   num_heads=8, addition_embed_type="text", addition_embed_type_num_heads=4, resnet_time_scale_shift="scale_shift")
    unet = UNet1DConditionModel(in_channels=c.in_channels, out_channels=c.out_channels, block_out_channels=c.block_out_channels,
                                layers_per_block=list(c.layers_per_block), norm_num_groups=c.norm_num_groups,
                                cross_attention_dim=c.cross_attention_dim, attention_head_dim=c.num_heads,
                                addition_embed_type=c.addition_embed_type, addition_embed_type_num_heads=c.addition_embed_type_num_heads,
                                resnet_time_scale_shift=c.resnet_time_scale_shift)
    unet.load_state_dict(make_state_dict(c, 0))
    unet = unet.to(dev).eval()
    voc = Vocos.from_state_dict(make_vocos_state_dict(0, "trained_like", dim=128, intermediate_dim=384, num_layers=2)).to(dev)
    g = torch.Generator().manual_seed(3)
    wavs = []
    for d in DURATIONS:
        n = int(d * SR)
        t = torch.arange(n) / SR
        wavs.append((0.3 * torch.sin(2 * torch.pi * (110 + 300 * torch.rand(1, generator=g)) * t) + 0.05 * torch.randn(n, generator=g)).float())
    prompt = (torch.randn((100, 70), generator=g) - 4.0).float()
    return (cv, pre, unet, voc), wavs, prompt


def _conversions(models, wavs, prompt, dev, group):
    """Default-x_T conversion after seed 1234, the generator state after it, the same with the x_T drawn by hand after the same
    seed, and convert_slices after seed 99."""
    from test_convert import _audio_data
    torch.manual_seed(1234)
    default = convert.convert_utterances(*models, wavs, SR, prompt, steps=STEPS, max_batch=4, group=group)
    state = torch.cuda.get_rng_state(dev)
    torch.manual_seed(1234)
    xs = [torch.randn((1, 100, convert.frame_plan(len(w), SR)["T"]), device=dev) for w in wavs]
    explicit = convert.convert_utterances(*models, wavs, SR, prompt, steps=STEPS, max_batch=4, x_T=xs, group=group)
    torch.manual_seed(99)
    sl = convert.convert_slices(*models, _audio_data(5), SR, prompt, pad_seconds=0.5, clip_seconds=1.0, linear_gradient=0.2,
                                steps=STEPS, max_batch=4, group=group)
    return dict(default=[a.cpu() for a in default], explicit=[a.cpu() for a in explicit], state=state.cpu(), slices=torch.from_numpy(sl))


def _convert_worker(rank, world, out_dir):
    dev = torch.device("cuda", torch.cuda.current_device())
    models, wavs, prompt = _chain(dev)
    res = _conversions(models, wavs, prompt, dev, dist.group.WORLD)
    res["backend"] = str(dist.get_backend())
    path = os.path.join(out_dir, f"rank{rank}.pt")
    torch.save(res, path)
    return path


@pytest.fixture(scope="module")
def sharded(tmp_path_factory):
    """The single-process results and those of each of 2 ranks."""
    dev = torch.device("cuda", 0)
    models, wavs, prompt = _chain(dev)
    one = _conversions(models, wavs, prompt, dev, None)
    backend = "nccl" if torch.cuda.device_count() >= 2 else "gloo"
    paths = _run(_convert_worker, 2, str(tmp_path_factory.mktemp("ranks")), backend=backend, timeout=600)
    assert all(p.endswith(".pt") for p in paths), paths
    ranks = [torch.load(p, weights_only=False) for p in paths]
    print(f"2 ranks over {ranks[0]['backend']}")
    return one, ranks


def _rel(a, b):
    a, b = a.double(), b.double()
    return ((a - b).norm() / b.norm()).item()


@pytest.mark.gpu
def test_sharded_utterances_match_the_single_process_call(sharded):
    one, ranks = sharded
    bad = []
    for r, res in enumerate(ranks):
        for key in ("default", "explicit"):
            got, want = res[key], one[key]
            assert len(got) == len(want)
            same = 0
            for i, (a, b) in enumerate(zip(got, want)):
                assert a.shape == b.shape, f"rank {r} {key} {i}: {tuple(a.shape)} vs {tuple(b.shape)}"
                assert torch.equal(a, ranks[0][key][i]), f"rank {r} {key} {i}: ranks return different results"
                same += torch.equal(a, b)
                if _rel(a, b) > 1e-4:
                    bad.append(f"rank {r} {key} utterance {i}: ||sharded - one|| / ||one|| {_rel(a, b):.2e}")
            print(f"rank {r} {key}: {same} of {len(want)} utterances bit-identical to the single-process call, worst "
                  f"||sharded - one|| / ||one|| {max(_rel(a, b) for a, b in zip(got, want)):.2e}")
    assert not bad, "\n".join(bad)


@pytest.mark.gpu
def test_sharded_default_x_T_and_generator_state_equal_the_single_process_call(sharded):
    one, ranks = sharded
    for r, res in enumerate(ranks):
        for i, (a, b) in enumerate(zip(res["default"], res["explicit"])):
            assert torch.equal(a, b), f"rank {r} utterance {i}: the default x_T is not the single-process draw"
        assert torch.equal(res["state"], one["state"]), f"rank {r}: the generator ends elsewhere than after the single-process call"


@pytest.mark.gpu
def test_sharded_convert_slices_matches_the_single_process_call(sharded):
    one, ranks = sharded
    for r, res in enumerate(ranks):
        a, b = res["slices"], one["slices"]
        assert a.dtype == torch.float64 and a.shape == b.shape
        print(f"rank {r}: convert_slices ||sharded - one|| / ||one|| {_rel(a, b):.2e}, bit-identical {torch.equal(a, b)}")
        assert _rel(a, b) <= 1e-4
