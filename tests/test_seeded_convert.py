"""Seeded DDPM / DDIM in the conversion chain and the server: each waveform's x_T and step noise drawn from its own seed.

CPU: without seeds DDPM / DDIM are still refused with ``convert._check_method``'s message; the seed, eta and step checks.
GPU: ``convert_utterances(noise_seeds=...)`` equals ``convert_batch`` of each waveform alone with its seed, bit for bit, at
max_batch 1 and 8; a server tick mixing UniPC, DPM-Solver++, DDIM (eta 0.5) and DDPM requests arriving at different ticks gives
each request that same result, and a request's audio is the same served alone; two ranks over gloo equal one GPU for both."""
import os

import pytest
import torch
import torch.distributed as dist

from ns2vc_b200 import convert, serve
from test_convert import SR
from test_serve import MAX_FRAMES, MAX_PROMPT, SLOTS, chain  # noqa: F401  (chain: the shared fixture)
from test_shard_convert import _run

SEEDS = [11, 12, 1 << 40, 14, (1 << 63) - 1, 16]
# the six requests' (method, steps, eta) and the ticks they arrive at
REQ = [("unipc", 6, 0.0), ("ddim", 10, 0.5), ("dpmsolver", 5, 0.0), ("ddpm", None, 0.0), ("ddim", 7, 0.0), ("unipc", 4, 0.0)]
ARRIVALS = {0: [0, 1], 2: [2, 3], 5: [4], 9: [5]}


# ----------------------------------------------------------------------------------------------------------------- CPU
def test_unseeded_ddpm_ddim_keep_the_refusal_and_seeded_arguments_are_checked():
    w, mel = torch.zeros(20000), torch.zeros(100, 30)
    for method in ("ddpm", "ddim"):
        with pytest.raises(ValueError) as want:
            convert._check_method(method, None)
        with pytest.raises(ValueError) as got:
            convert.convert_utterances(None, None, None, None, [w], SR, mel, method=method)
        assert str(got.value) == str(want.value)
        srv = serve.ConversionServer(None, None, None, None, slots=2, max_frames=100, max_prompt_frames=40)
        with pytest.raises(ValueError) as got:
            srv.submit(w, SR, mel, method=method)
        assert str(got.value) == str(want.value)
    assert convert._check_method("ddpm", None, seeded=True) == 1000 and convert._check_method("ddim", None, seeded=True) == 100
    assert convert._check_method("ddim", 7, seeded=True) == 7 and convert._check_method("unipc", None, seeded=True) == 30
    with pytest.raises(ValueError):
        convert._check_method("ddpm", 10, seeded=True)
    for method, kw in (("ddim", dict(noise_seeds=[1, 2])), ("ddim", dict(noise_seeds=[-1])), ("ddpm", dict(noise_seeds=[1 << 63])),
                       ("ddim", dict(noise_seeds=[1], eta=1.5)), ("ddim", dict(noise_seeds=[1], eta=-0.5)),
                       ("ddpm", dict(noise_seeds=[1], eta=0.5)), ("unipc", dict(noise_seeds=[1], eta=0.5))):
        with pytest.raises(ValueError):
            convert.convert_utterances(None, None, None, None, [w], SR, mel, method=method, **kw)
    srv = serve.ConversionServer(None, None, None, None, slots=2, max_frames=100, max_prompt_frames=40)
    for kw in (dict(seed=-1, method="ddim"), dict(seed=1 << 63, method="ddpm"), dict(seed=1, method="ddim", eta=2.0),
               dict(seed=1, method="unipc", eta=0.5), dict(seed=1, method="ddpm", steps=50)):
        with pytest.raises(ValueError):
            srv.submit(w, SR, mel, **kw)
    assert srv.table.idle


# ----------------------------------------------------------------------------------------------------------------- GPU
def _alone(models, wav, prompt, seed, method, steps, eta):
    r = convert.convert_batch(*models, [wav], SR, [prompt], None, method, steps, noise_seeds=[seed], eta=eta)
    return r["latent"][0].cpu(), r["audio"][0].cpu()


@pytest.mark.gpu
def test_seeded_conversion_equals_each_waveform_alone(chain):
    models, wavs, prompt, _ = chain
    for method, steps, eta, batches in (("ddim", 10, 0.5, (1, 8)), ("ddpm", None, 0.0, (8,))):
        alone = [_alone(models, w, prompt, s, method, steps, eta)[1] for w, s in zip(wavs, SEEDS)]
        for mb in batches:
            got = convert.convert_utterances(*models, wavs, SR, prompt, method=method, steps=steps, max_batch=mb, noise_seeds=SEEDS,
                                             eta=eta)
            bad = [i for i in range(len(wavs)) if not torch.equal(got[i].cpu(), alone[i])]
            assert not bad, f"{method} max_batch={mb}: waveforms {bad} differ from their own conversion"


def _serve_script(srv, wavs, prompt, submit=True, only=None):
    """Serves REQ on ARRIVALS (``only``: just that request, at tick 0), each with its seed.  Returns
    ({request: audio}, {request: latent})."""
    arrivals = ARRIVALS if only is None else {0: [only]}
    req, res, lat = {}, {}, {}
    while True:
        if submit:
            for i in arrivals.get(srv.ticks, ()):
                m, s, eta = REQ[i]
                req[srv.submit(wavs[i], SR, prompt, method=m, steps=s, seed=SEEDS[i], eta=eta)] = i
        done = srv.tick()
        for tk, v in done.items():
            res[req[tk]] = v.cpu() if isinstance(v, torch.Tensor) else v
        lat.update({req[tk]: v.cpu() for tk, v in srv.last_latents.items()})
        idle = srv._idle if srv.world > 1 else srv.table.idle
        if srv.ticks > max(arrivals) and idle:
            return res, lat


@pytest.mark.gpu
def test_server_tick_with_seeded_ddpm_ddim_rows_equals_each_request_alone(chain):
    models, wavs, prompt, _ = chain
    kw = dict(slots=SLOTS, max_frames=MAX_FRAMES, max_prompt_frames=MAX_PROMPT, method="dpmsolver", steps=5)
    res, lat = _serve_script(serve.ConversionServer(*models, **kw), wavs, prompt)
    assert sorted(res) == list(range(len(REQ)))
    bad = []
    for i, (m, s, eta) in enumerate(REQ):
        la, aa = _alone(models, wavs[i], prompt, SEEDS[i], m, s, eta)
        if not (torch.equal(lat[i], la) and torch.equal(res[i], aa)):
            bad.append(f"request {i} {REQ[i]}: max|latent diff| {(lat[i] - la).abs().max().item():.3e}")
    assert not bad, "\n".join(bad)
    for i in (1, 3):                                          # the DDIM and DDPM requests served alone
        solo, _ = _serve_script(serve.ConversionServer(*models, **kw), wavs, prompt, only=i)
        assert torch.equal(solo[i], res[i]), f"request {i} alone differs from request {i} among others"


def _gpu_worker(rank, world, out_dir):
    from test_shard_convert import _chain
    dev = torch.device("cuda", torch.cuda.current_device())
    models, wavs, prompt = _chain(dev)
    out = {"rank": rank}
    conv = convert.convert_utterances(*models, wavs, SR, prompt, method="ddim", steps=10, eta=0.5, max_batch=2,
                                      noise_seeds=SEEDS, group=dist.group.WORLD)
    kw = dict(slots=2, max_frames=400, max_prompt_frames=80, method="dpmsolver", steps=5)
    res, lat = _serve_script(serve.ConversionServer(*models, group=dist.group.WORLD, **kw), wavs, prompt, submit=rank == 0)
    if rank == 0:
        one = convert.convert_utterances(*models, wavs, SR, prompt, method="ddim", steps=10, eta=0.5, max_batch=2, noise_seeds=SEEDS)
        out["convert"] = [i for i in range(len(wavs)) if not torch.equal(conv[i].cpu(), one[i].cpu())]
        one_res, one_lat = _serve_script(serve.ConversionServer(*models, **dict(kw, slots=2 * world)), wavs, prompt)
        out["serve"] = [i for i in range(len(REQ)) if not (torch.equal(res[i], one_res[i]) and torch.equal(lat[i], one_lat[i]))]
    else:
        out["empty"] = res == {} and lat == {}
        out["convert_len"] = len(conv)
    path = os.path.join(out_dir, f"rank{rank}.pt")
    torch.save(out, path)
    return path


@pytest.mark.gpu
def test_two_ranks_with_seeds_equal_one_gpu(tmp_path):
    paths = _run(_gpu_worker, 2, str(tmp_path), backend="gloo", timeout=900)
    r0, r1 = [torch.load(p, weights_only=False) for p in paths]
    print(f"2 ranks over gloo: {r0} {r1}")
    assert r0["convert"] == [], f"waveforms {r0['convert']} differ from the one-GPU conversion"
    assert r0["serve"] == [], f"requests {r0['serve']} differ from the one-GPU server"
    assert r1["empty"] is True and r1["convert_len"] == len(SEEDS)
