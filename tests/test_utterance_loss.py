"""Each utterance's own training objective: ``loss.utterance_losses`` / ``batch_utterance_losses`` / ``mse_rows_ragged`` against
``NaturalSpeech2.forward`` (reference model.py:706-734) on unpadded B = 1 batches.

CPU: the oracle reproduces tests/golden/utterance_loss.pt (written by the unmodified reference, oracle/make_golden_utterance_loss.py),
argument errors, and the reduction's host checks.  GPU: every utterance matches the fixture in one ragged batch and in batches of
two; values do not depend on the batching; the ragged reduction is exact, deterministic and blind to its padding; NaN in the
packed inputs' padding changes nothing; a grid of K timesteps equals K calls; the default draws are those of the one-by-one
``diffusion_loss`` loop; the padded objective and the samplers are undisturbed; two ranks return the one-GPU result."""
import os
import types

import pytest
import torch

from ns2vc_b200 import coefs
from ns2vc_b200.arch import ns2vc_denoiser_config
from ns2vc_b200.synth import make_pre_state_dict, make_state_dict, make_utterance_loss_inputs, state_dict_checksum

LOSS_RTOL = 5e-5                     # the bound of tests/test_train_loss.py: GPU loss / row MSE against the fp64 oracle
BATCH_RTOL = 1e-3                    # one utterance in two ragged batches: the ragged denoiser's row tolerance, carried to its MSE
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
PRE_CFG = {"phoneme_encoder": dict(in_channels=256, hidden_channels=256, out_channels=256, n_layers=6, p_dropout=0.2),
           "prompt_encoder": dict(in_channels=100, hidden_channels=256, out_channels=256, n_layers=6, p_dropout=0.2)}


def bits(x):
    return x.contiguous().view(torch.int32)


def fixture_inputs(g):
    """The fixture's inputs, regenerated from its seeds and checked against its checksums."""
    out = []
    for i, u in enumerate(g["utterances"]):
        inp = make_utterance_loss_inputs(u["T"], u["S"], u["seed"])
        assert state_dict_checksum(inp) == u["inputs_checksum"], f"utterance {i}: regenerated inputs differ from the fixture's"
        out.append(inp)
    return out


def fixture_items(g):
    ins = fixture_inputs(g)
    return [(v["c"], v["spec"], v["refer"]) for v in ins], torch.tensor([u["t"] for u in g["utterances"]]), [v["noise"] for v in ins]


def rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return ((a - b).abs() / b.abs()).max().item()


# ------------------------------------------------------------------------------------------------------------------- CPU
def test_oracle_reproduces_the_per_utterance_fixture(gold):
    from oracle import loss_oracle
    g = gold("utterance_loss.pt")
    sd_u, sd_p = make_state_dict(ns2vc_denoiser_config(), seed=0), make_pre_state_dict(PRE_CFG, seed=0)
    assert state_dict_checksum(sd_u) == g["unet_checksum"] and state_dict_checksum(sd_p) == g["pre_checksum"]
    assert torch.equal(g["buffers"]["loss_weight"], coefs.loss_buffers(1000)["loss_weight"])
    us = g["utterances"]
    assert {0, 999} <= {u["t"] for u in us} and len({u["S"] for u in us}) == len(us)
    for i, (u, v) in enumerate(zip(us, fixture_inputs(g))):
        T, S = u["T"], u["S"]
        assert v["spec"].shape == (100, T) and v["refer"].shape == (100, S)
        o = loss_oracle.diffusion_loss(sd_p, sd_u, ns2vc_denoiser_config(), v["c"][None], v["refer"][None], v["spec"][None],
                                       torch.tensor([T]), torch.tensor([S]), torch.tensor([u["t"]]), v["noise"][None])
        assert (o["model_out"][0] - u["model_out"]).abs().max().item() <= 2e-5, i
        assert abs(o["loss"].item() - u["loss"].item()) <= 1e-6 * abs(u["loss"].item()), i
        # B = 1: forward's product of means is weight x MSE, and the MSE is over the utterance's own 100 x T_i elements
        assert abs((u["weight"].double() * u["mse64"]).item() - u["loss"].item()) <= 1e-5 * abs(u["loss"].item()), i


def _cpu_models():
    """A denoiser left on the CPU (20 latent + 16 content channels) and a stand-in for the encoders, which are never reached."""
    from ns2vc_b200.unet import UNet1DConditionModel
    unet = UNet1DConditionModel(in_channels=36, out_channels=20, block_out_channels=(32, 64, 64, 96), norm_num_groups=8,
                                cross_attention_dim=16, attention_head_dim=8)
    return types.SimpleNamespace(infer=None), unet


def test_argument_errors():
    from ns2vc_b200 import api
    from ns2vc_b200.loss import utterance_losses
    assert api.utterance_losses is utterance_losses
    pre, unet = _cpu_models()
    items = [(torch.zeros(16, 12), torch.zeros(20, 12), torch.zeros(20, 6)), (torch.zeros(16, 5), torch.zeros(20, 5), torch.zeros(20, 3))]
    with pytest.raises(RuntimeError, match="no CPU path"):
        utterance_losses(pre, unet, items)
    t = torch.tensor([0, 999])
    bad = [
        ([], {}),                                                                              # empty
        ([items[0][:2]], {}),                                                                  # not a triple
        ([(torch.zeros(16, 12), torch.zeros(19, 12), torch.zeros(20, 6))], {}),                # spec channels
        ([(torch.zeros(16, 11), torch.zeros(20, 12), torch.zeros(20, 6))], {}),                # c frames
        ([(torch.zeros(16, 0), torch.zeros(20, 0), torch.zeros(20, 6))], {}),                  # T_i = 0
        ([(torch.zeros(16, 4), torch.zeros(20, 4), torch.zeros(20, 0))], {}),                  # S_i = 0
        ([(torch.zeros(16, 4), torch.zeros(20, 4), torch.zeros(20))], {}),                     # refer not 2-D
        (items + [(torch.zeros(8, 4), torch.zeros(20, 4), torch.zeros(20, 3))], {}),           # channel counts differ
        (items, dict(t=t, t_grid=[0, 5])),                                                     # both t and t_grid
        (items, dict(t=torch.tensor([0, 1000]))),                                              # t outside [0, timesteps)
        (items, dict(t=torch.tensor([-1, 5]))),
        (items, dict(t=torch.tensor([0, 10]), timesteps=10)),
        (items, dict(t=torch.tensor([0, 1], dtype=torch.int32))),                              # dtype
        (items, dict(t=torch.tensor([0, 1, 2]))),                                              # [N]
        (items, dict(t_grid=[])),
        (items, dict(t_grid=[0, 1000])),
        (items, dict(noise=[torch.zeros(20, 12)])),                                            # one per utterance
        (items, dict(noise=[torch.zeros(20, 12), torch.zeros(20, 6)])),                        # [100, T_i]
        (items, dict(max_batch=0)),
        (items, dict(min_snr_gamma=0.0)),
        (items, dict(timesteps=0)),
    ]
    for its, kw in bad:
        with pytest.raises(ValueError):
            utterance_losses(pre, unet, its, **kw)


def test_ragged_reduction_host_checks():
    from ns2vc_b200.loss import mse_rows_ragged
    K, B, C, T = 2, 3, 4, 10
    out, target, t = torch.zeros(K, B, C, T), torch.zeros(B, C, T), torch.zeros(K, B, dtype=torch.int64)
    ln = [10, 1, 7]
    bad = [
        (torch.zeros(B, C, T), target, ln, t),                          # out not [K, B, C, T]
        (out, torch.zeros(B, C, T + 1), ln, t),                         # target shape
        (out, torch.zeros(K + 1, B, C, T), ln, t),
        (out, target, ln, torch.zeros(K, B, dtype=torch.int32)),        # t dtype
        (out, target, ln, torch.zeros(B, dtype=torch.int64)),           # t shape
        (out, target, [10, 0, 7], t),                                   # lengths outside [1, T]
        (out, target, [10, 11, 7], t),
        (out, target, [10, 7], t),                                      # B lengths
    ]
    for a in bad:
        with pytest.raises(ValueError):
            mse_rows_ragged(*a)
    with pytest.raises(ValueError, match="CUDA"):
        mse_rows_ragged(out, target, ln, t)


# ------------------------------------------------------------------------------------------------------------------- GPU
@pytest.fixture(scope="module")
def models():
    from ns2vc_b200.pre_model import Pre_model
    from ns2vc_b200.unet import UNet1DConditionModel
    unet = UNet1DConditionModel(in_channels=356, out_channels=100, block_out_channels=(128, 256, 384, 512), norm_num_groups=8,
                                cross_attention_dim=256, attention_head_dim=8, addition_embed_type="text", resnet_time_scale_shift="scale_shift")
    unet.load_state_dict(make_state_dict(ns2vc_denoiser_config(), seed=0))
    pre = Pre_model(PRE_CFG)
    pre.load_state_dict(make_pre_state_dict(PRE_CFG, seed=0))
    return pre.cuda().eval(), unet.cuda().eval()


@pytest.mark.gpu
@pytest.mark.parametrize("max_batch", [8, 2])
def test_each_utterance_reproduces_the_reference(gold, models, max_batch):
    from ns2vc_b200.loss import utterance_losses
    pre, unet = models
    g = gold("utterance_loss.pt")
    items, t, noise = fixture_items(g)
    r = utterance_losses(pre, unet, items, t=t, noise=noise, max_batch=max_batch)
    assert r.loss.shape == (5,) and r.mse.shape == (5,) and r.t.tolist() == t.tolist()
    want = torch.stack([u["loss"] for u in g["utterances"]])
    mse64 = torch.stack([u["mse64"] for u in g["utterances"]])
    w = torch.stack([u["weight"] for u in g["utterances"]])
    e_loss, e_mse = rel(r.loss, want), rel(r.mse, mse64)
    print(f"[max_batch {max_batch}] loss rel {e_loss:.2e}, mse rel {e_mse:.2e} (vs fp64)")
    assert e_loss <= LOSS_RTOL and e_mse <= LOSS_RTOL
    assert rel(r.loss, r.mse.cpu() * w) <= 1e-6
    r5 = utterance_losses(pre, unet, items, t=t, noise=noise, max_batch=max_batch, min_snr_gamma=5.0)
    assert torch.equal(bits(r5.mse), bits(r.mse)) and rel(r5.loss, r.mse.cpu() * w.clamp(max=5.0)) <= 1e-6


@pytest.mark.gpu
def test_values_do_not_depend_on_the_batching(gold, models):
    from ns2vc_b200.loss import utterance_losses
    pre, unet = models
    items, t, noise = fixture_items(gold("utterance_loss.pt"))
    base = utterance_losses(pre, unet, items, t=t, noise=noise, max_batch=1)      # each utterance alone
    worst = 0.0
    for mb in (2, 3, 8):
        r = utterance_losses(pre, unet, items, t=t, noise=noise, max_batch=mb)
        worst = max(worst, rel(r.loss, base.loss), rel(r.mse, base.mse))
        assert torch.equal(bits(r.loss), bits(utterance_losses(pre, unet, items, t=t, noise=noise, max_batch=mb).loss)), mb
    # other batch partners: two longer utterances join, the list is reversed
    g = torch.Generator().manual_seed(11)
    extra = [(torch.randn(256, T, generator=g), torch.randn(100, T, generator=g), torch.randn(100, S, generator=g)) for T, S in ((311, 90), (257, 12))]
    extra_noise = [torch.randn(100, it[1].shape[1], generator=g) for it in extra]
    r = utterance_losses(pre, unet, extra + items[::-1], t=torch.cat([torch.tensor([5, 600]), t.flip(0)]),
                         noise=extra_noise + noise[::-1], max_batch=4)
    worst = max(worst, rel(r.loss[2:].flip(0), base.loss), rel(r.mse[2:].flip(0), base.mse))
    print(f"worst rel difference to the utterance alone over the batchings: {worst:.2e}")
    assert worst <= BATCH_RTOL


@pytest.mark.gpu
def test_ragged_reduction_is_exact_deterministic_and_blind_to_padding():
    from ns2vc_b200.loss import mse_rows, mse_rows_ragged
    g = torch.Generator(device="cuda").manual_seed(3)
    C, K = 100, 2
    lens = [1, 81, 82, 203, 300]                                    # C * T_b from 100 to 30 000: one to four chunks
    tt = torch.tensor([[0, 999, 500, 37, 1], [10, 10, 10, 10, 10]], device="cuda")
    rows = [(torch.randn(K, C, T, device="cuda", generator=g) * 3, torch.randn(C, T, device="cuda", generator=g)) for T in lens]
    ref64 = [((o.double() - x.double()[None]) ** 2).reshape(K, -1).mean(-1) for o, x in rows]
    w = coefs.loss_buffers(1000)["loss_weight"].cuda().double()

    def packed(order, T, fill):
        B = len(order)
        out = torch.full((K, B, C, T), fill, device="cuda")
        tgt = torch.full((B, C, T), fill, device="cuda")
        for j, i in enumerate(order):
            out[:, j, :, :lens[i]] = rows[i][0]
            tgt[j, :, :lens[i]] = rows[i][1]
        return out, tgt, [lens[i] for i in order], tt[:, order].contiguous()

    first = {}
    for order, T, fill in (([0, 1, 2, 3, 4], 300, 0.0), ([4, 3, 2, 1, 0], 300, float("nan")), ([2, 0], 90, float("inf")),
                           ([3, 1, 3], 1000, float("nan")), ([1], 81, 0.0), ([4, 2], 4099, -float("inf"))):
        out, tgt, ln, tk = packed(order, T, fill)
        a = mse_rows_ragged(out, tgt, ln, tk)
        b = mse_rows_ragged(out, tgt[None].expand(K, -1, -1, -1).contiguous(), ln, tk)    # a [K, B, C, T] target
        ws = torch.full((1 << 20,), 0xFF, dtype=torch.uint8, device="cuda")
        c = mse_rows_ragged(out, tgt, ln, tk, ws=ws)
        for x, y in zip(a, b):
            assert torch.equal(bits(x), bits(y))
        for x, y in zip(a, c):
            assert torch.equal(bits(x), bits(y))
        for j, i in enumerate(order):
            got = torch.stack([a[0][:, j], a[1][:, j]])
            assert torch.isfinite(got).all()
            if i in first:
                assert torch.equal(bits(got), bits(first[i])), (order, T, i)       # same bits in any batch, at any row, any T
            else:
                first[i] = got
                assert rel(a[0][:, j], ref64[i]) <= 1e-6 and rel(a[1][:, j], ref64[i] * w[tk[:, j]]) <= 1e-6
                # and the padded reduction of the unpadded row gives the same bits
                o1, t1, _, k1 = packed([i], lens[i], 0.0)
                p = mse_rows(o1, t1, k1)
                assert torch.equal(bits(p[0][:, 0]), bits(got[0])) and torch.equal(bits(p[1][:, 0]), bits(got[1]))
    assert len(first) == len(lens)


@pytest.mark.gpu
def test_nan_in_the_padding_of_packed_inputs_changes_nothing(gold, models):
    from ns2vc_b200.loss import batch_utterance_losses
    pre, unet = models
    items, t, noise = fixture_items(gold("utterance_loss.pt"))
    tl = [it[1].shape[1] for it in items]
    sl = [it[2].shape[1] for it in items]
    B, T, S = len(items), max(tl), max(sl)

    def pack(fill):
        c = torch.full((B, 256, T), fill)
        spec = torch.full((B, 100, T), fill)
        refer = torch.full((B, 100, S), fill)
        nz = torch.full((B, 100, T), fill)
        for b, (ci, si, ri) in enumerate(items):
            c[b, :, :tl[b]], spec[b, :, :tl[b]], refer[b, :, :sl[b]], nz[b, :, :tl[b]] = ci, si, ri, noise[b]
        return [v.cuda() for v in (c, refer, spec, nz)]

    tk = t[None].cuda()
    c, refer, spec, nz = pack(0.0)
    clean = batch_utterance_losses(pre, unet, c, refer, spec, tl, sl, tk, nz)
    c, refer, spec, nz = pack(float("nan"))
    dirty = batch_utterance_losses(pre, unet, c, refer, spec, tl, sl, tk, nz)
    for a, b in zip(clean, dirty):
        assert torch.isfinite(a).all() and torch.equal(bits(a), bits(b))


@pytest.mark.gpu
def test_a_grid_of_k_timesteps_equals_k_calls(gold, models):
    from ns2vc_b200.loss import utterance_losses
    pre, unet = models
    items, _, noise = fixture_items(gold("utterance_loss.pt"))
    grid = [0, 3, 500, 999]
    prof = utterance_losses(pre, unet, items, t_grid=grid, noise=noise, max_batch=3)
    assert prof.loss.shape == (4, 5) and prof.mse.shape == (4, 5) and prof.t.tolist() == [[v] * 5 for v in grid]
    for k, v in enumerate(grid):
        one = utterance_losses(pre, unet, items, t=torch.full((5,), v), noise=noise, max_batch=3)
        assert torch.equal(bits(prof.loss[k]), bits(one.loss)) and torch.equal(bits(prof.mse[k]), bits(one.mse)), v


@pytest.mark.gpu
def test_default_draws_are_those_of_the_one_by_one_loop(gold, models):
    from ns2vc_b200.loss import diffusion_loss, utterance_losses
    pre, unet = models
    items, _, _ = fixture_items(gold("utterance_loss.pt"))
    torch.manual_seed(23)
    r = utterance_losses(pre, unet, items, max_batch=2)
    state = torch.cuda.get_rng_state()
    torch.manual_seed(23)
    loop_t, loop_loss, loop_mse = [], [], []
    for c, spec, refer in items:
        data = (c[None].cuda(), refer[None].cuda(), None, spec[None].cuda(), None, torch.tensor([spec.shape[1]]),
                torch.tensor([refer.shape[1]]), None)
        one = diffusion_loss(pre, unet, data)
        loop_t.append(int(one.t[0]))
        loop_loss.append(one.loss)
        loop_mse.append(one.loss_row[0])
    assert torch.equal(torch.cuda.get_rng_state(), state)
    assert r.t.tolist() == loop_t
    e = max(rel(r.loss, torch.stack(loop_loss)), rel(r.mse, torch.stack(loop_mse)))
    print(f"ragged call vs the diffusion_loss loop: worst rel {e:.2e}")
    assert e <= 2 * LOSS_RTOL
    # the same draws by hand give the same values bit for bit
    torch.manual_seed(23)
    t, noise = [], []
    for _, spec, _ in items:
        t.append(torch.randint(0, 1000, (1,), device="cuda").long())
        noise.append(torch.randn_like(spec[None].cuda())[0])
    explicit = utterance_losses(pre, unet, items, t=torch.cat(t).cpu(), noise=noise, max_batch=8)
    assert torch.equal(bits(explicit.loss), bits(r.loss)) and torch.equal(bits(explicit.mse), bits(r.mse))


@pytest.mark.gpu
def test_padded_objective_and_samplers_are_undisturbed(gold, models):
    """diffusion_loss, a padded sampler and a ragged sampler whose session shape is that of the utterance batch, before and after
    utterance_losses: bit-identical results (four sampler runs, so captured loops are replayed around the calls as well)."""
    from ns2vc_b200 import api
    from ns2vc_b200.loss import diffusion_loss, utterance_losses
    pre, unet = models
    k = gold("train_loss.pt")["cases"]["drawn"]
    data = (k["c"].cuda(), k["refer"].cuda(), None, k["spec"].cuda(), None, k["lengths"].cuda(), k["refer_lengths"].cuda(), None)
    items, t, noise = fixture_items(gold("utterance_loss.pt"))
    gen = torch.Generator().manual_seed(4)
    xT = torch.randn(tuple(k["spec"].shape), generator=gen).cuda()
    s_items = [(torch.randn(100, it[1].shape[1], generator=gen), torch.randn(it[1].shape[1], 256, generator=gen),
                torch.randn(it[2].shape[1], 256, generator=gen)) for it in items]          # (B, T, S) of the utterance batch

    def run():
        a = diffusion_loss(pre, unet, data, t=k["t"].cuda(), noise=k["noise"].cuda())
        b = api.sample_from_features(pre, unet, xT, data[0], data[1], data[5], data[6], steps=6, method="dpmsolver")
        c = api.sample_utterances(unet, s_items, steps=6, method="dpmsolver", max_batch=8)
        return [a.loss, a.model_out, b] + c
    first = run()
    want = utterance_losses(pre, unet, items, t=t, noise=noise, max_batch=8)
    for i in range(3):
        got = utterance_losses(pre, unet, items, t=t, noise=noise, max_batch=8)
        assert torch.equal(bits(got.loss), bits(want.loss)), f"run {i}"
        again = run()
        assert all(torch.equal(bits(x), bits(y)) for x, y in zip(again, first)), f"run {i}"


# ------------------------------------------------------------------------------------------------------- several GPUs
def _rank_worker(rank, world, out_dir):
    from ns2vc_b200 import loss
    import torch.distributed as dist
    dev = torch.device("cuda", torch.cuda.current_device())
    from ns2vc_b200.pre_model import Pre_model
    from ns2vc_b200.unet import UNet1DConditionModel
    unet = UNet1DConditionModel(in_channels=356, out_channels=100, block_out_channels=(128, 256, 384, 512), norm_num_groups=8,
                                cross_attention_dim=256, attention_head_dim=8, addition_embed_type="text", resnet_time_scale_shift="scale_shift")
    unet.load_state_dict(make_state_dict(ns2vc_denoiser_config(), seed=0))
    pre = Pre_model(PRE_CFG)
    pre.load_state_dict(make_pre_state_dict(PRE_CFG, seed=0))
    pre, unet = pre.to(dev).eval(), unet.to(dev).eval()
    items, t, noise = fixture_items(torch.load(os.path.join(GOLD, "utterance_loss.pt"), map_location="cpu",
                                                   weights_only=False))
    res = _rank_results(pre, unet, items, t, noise, dist.group.WORLD)
    orig = loss.batch_utterance_losses

    def failing(*a, **kw):
        if dist.get_rank() == 1:
            raise AssertionError("rank 1 fails on purpose")
        return orig(*a, **kw)
    loss.batch_utterance_losses = failing
    try:
        loss.utterance_losses(pre, unet, items, t=t, noise=noise, max_batch=2, group=dist.group.WORLD)
        res["failure"] = "no error"
    except RuntimeError as e:
        res["failure"] = str(e)
    finally:
        loss.batch_utterance_losses = orig
    res["backend"] = str(dist.get_backend())
    path = os.path.join(out_dir, f"rank{rank}.pt")
    torch.save(res, path)
    return path


def _rank_results(pre, unet, items, t, noise, group):
    from ns2vc_b200.loss import utterance_losses
    explicit = utterance_losses(pre, unet, items, t=t, noise=noise, max_batch=2, group=group)
    grid = utterance_losses(pre, unet, items, t_grid=[0, 999, 300], noise=noise, max_batch=2, group=group)
    torch.manual_seed(77)
    drawn = utterance_losses(pre, unet, items, max_batch=2, group=group)
    return dict(explicit=explicit.loss.cpu(), explicit_mse=explicit.mse.cpu(), grid=grid.loss.cpu(), drawn=drawn.loss.cpu(),
                drawn_t=drawn.t.cpu(), state=torch.cuda.get_rng_state().cpu())


@pytest.mark.gpu
def test_two_ranks_return_the_one_gpu_result(gold, models, tmp_path):
    """Two ranks over NCCL on two GPUs, or over gloo with both ranks on cuda:0 when there is one."""
    from test_shard_convert import _run
    pre, unet = models
    items, t, noise = fixture_items(gold("utterance_loss.pt"))
    one = _rank_results(pre, unet, items, t, noise, None)
    backend = "nccl" if torch.cuda.device_count() >= 2 else "gloo"
    paths = _run(_rank_worker, 2, str(tmp_path), backend=backend, timeout=600)
    assert all(p.endswith(".pt") for p in paths), paths
    for r, p in enumerate(paths):
        res = torch.load(p, weights_only=False)
        print(f"rank {r} over {res['backend']}")
        for key in ("explicit", "explicit_mse", "grid", "drawn", "drawn_t", "state"):
            assert torch.equal(res[key], one[key]), f"rank {r}: {key} differs from the one-GPU call"
        assert res["failure"].startswith("sharded run failed on rank(s) [1]"), f"rank {r}: {res['failure']}"
