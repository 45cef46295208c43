"""Row-scoped conditioning of a ragged denoiser program: ``ns2vc_unet_prepare_cond_rows`` and ``ns2vc_unet_time_table_rows``.

A ragged program is prepared in full; some rows then get new content, prompts and lengths and only they are prepared again.
Every row's ``forward_film`` output must equal, bit for bit, the output after a fresh full prepare of the same inputs; the
other rows must equal their outputs from before the change; the FiLM rows of the listed entries must equal the full table
there, and every other FiLM row must keep the poison written before the call.  The small configuration of ``test_serve.py``
and the flagship denoiser run at B = 4, and the flagship at the server's geometry (B = 8, T = 1024, S = 512) with the last
row listed.  CPU: the argument checks run without touching a device."""
import pytest
import torch

from ns2vc_b200 import _lib

K = 3


def _cfg(name):
    from ns2vc_b200.arch import UNetConfig, ns2vc_denoiser_config
    if name == "tiny":
        return UNetConfig(in_channels=132, out_channels=100, block_out_channels=(32, 64, 64, 96), norm_num_groups=8, cross_attention_dim=32,
                          num_heads=8, addition_embed_type="text", addition_embed_type_num_heads=4, resnet_time_scale_shift="scale_shift")
    return ns2vc_denoiser_config()


def test_rows_signatures():
    """The two entries take a host row list: ctypes must be told so, or a Python list would not convert."""
    import ctypes as C
    for name in ("ns2vc_unet_prepare_cond_rows", "ns2vc_unet_time_table_rows"):
        assert C.POINTER(C.c_int) in _lib.SIGNATURES[name][1], name


@pytest.mark.gpu
@pytest.mark.parametrize("name,B,T,S,rows", [("tiny", 4, 160, 48, [3, 1]), ("full", 4, 256, 48, [3, 1]),
                                             ("full", 8, 1024, 512, [7, 2, 5])])   # (the server's geometry, the last row listed)
def test_prepare_cond_rows_equals_a_full_prepare(name, B, T, S, rows):
    from ns2vc_b200.fused import DenoiserSession
    from test_gpu_parity import make_unet
    cfg = _cfg(name)
    unet, _ = make_unet(cfg)
    keep = [b for b in range(B) if b not in rows]
    Cl, Cc, xd = unet.latent_channels, cfg.in_channels - unet.latent_channels, cfg.cross_attention_dim
    g = torch.Generator(device="cuda").manual_seed(7)
    rnd = lambda *shape: torch.randn(shape, device="cuda", generator=g)
    content, prompt = rnd(B, Cc, T), rnd(B, S, xd)
    clen = [T if b == 0 else max(1, (T * (37 * b % 29 + 1)) // 30) for b in range(B)]
    plen = [S if b == 0 else max(1, (S * (17 * b % 13 + 1)) // 14) for b in range(B)]
    sess = DenoiserSession(unet, content, prompt, None, T=T, content_lengths=clen, prompt_lengths=plen)
    L, h = _lib.lib(), sess.h
    fw = int(L.ns2vc_unet_film_width(h))
    n_table = int(L.ns2vc_unet_time_table_floats(h, K * B))
    tvals = (torch.rand((K, B), device="cuda", generator=g) * 900 + 10).contiguous()
    x = rnd(B, Cl, T)

    def film_rows(table):
        return table[:K * B * fw].view(K, B, fw)

    def forward(table, k=1):
        out = torch.full((B, unet.cfg.out_channels, T), 3.0, device="cuda")
        sess.forward(x, None, out, film_rows=film_rows(table)[k].contiguous())
        torch.cuda.synchronize()
        return out

    sess.prepare()
    table = torch.empty(n_table, device="cuda")
    sess.time_table(tvals, table)
    before = forward(table)

    # new inputs and lengths for the listed rows; the others keep theirs (their input tensors are rewritten with the same values)
    for j, b in enumerate(rows):
        content[b], prompt[b] = rnd(Cc, T), rnd(S, xd)
        clen[b], plen[b] = (T, 5) if j == 0 else (max(1, clen[b] // 2 + 3), max(1, S - plen[b] + 1))
    sess.content.copy_(content)
    sess.prompt.copy_(prompt)
    sess.clen.copy_(torch.tensor(clen))
    sess.plen.copy_(torch.tensor(plen))
    sess.prepare_rows(rows)
    film_rows(table)[:, rows] = float("nan")           # the FiLM rows time_table_rows must rewrite
    poison = table.clone()
    film_rows(poison)[:, keep] = -7.25                 # the FiLM rows it must leave alone
    sess.time_table_rows(tvals, table, rows)
    sess.time_table_rows(tvals, poison, rows)
    got = [forward(table, k) for k in range(K)]

    sess.prepare()                                     # a fresh full prepare of the same inputs
    full = torch.empty(n_table, device="cuda")
    sess.time_table(tvals, full)
    want = [forward(full, k) for k in range(K)]
    torch.cuda.synchronize()

    for k in range(K):
        assert torch.equal(got[k], want[k]), f"{name}, step {k}: the row-prepared forward differs from the full prepare"
    assert torch.equal(got[1][keep], before[keep]), f"{name}: untouched rows changed"
    assert not any(torch.equal(got[1][b], before[b]) for b in rows), "a listed row did not change"
    for k in range(K):
        assert torch.equal(film_rows(poison)[k, rows], film_rows(full)[k, rows]), f"{name}, step {k}: listed FiLM rows"
        assert bool((film_rows(poison)[k, keep] == -7.25).all()), f"{name}, step {k}: an unlisted FiLM row was written"
    assert torch.equal(film_rows(table), film_rows(full))

    # every row listed: the full program, the same bytes; no row listed: nothing
    sess.prepare_rows(list(range(B)))
    sess.prepare_rows([])
    assert torch.equal(forward(full), want[1])


@pytest.mark.gpu
def test_prepare_cond_rows_refusals():
    B, S = 4, 48
    from ns2vc_b200.fused import DenoiserSession
    from test_gpu_parity import make_unet
    unet, _ = make_unet(_cfg("tiny"))
    T, xd = 64, 32
    content, prompt = torch.zeros((B, 32, T), device="cuda"), torch.zeros((B, S, xd), device="cuda")
    sess = DenoiserSession(unet, content, prompt, None, T=T, content_lengths=[T] * B, prompt_lengths=[S] * B)
    with pytest.raises(RuntimeError, match="prepare"):
        sess.prepare_rows([1])                         # nothing prepared yet
    sess.prepare()
    for rows, msg in (([4], "out of range"), ([-1], "out of range"), ([2, 2], "twice"), ([0, 1, 2, 3, 0], "rows of a batch")):
        with pytest.raises(_lib.Ns2vcError, match=msg):
            sess.prepare_rows(rows)
        table = torch.empty(int(_lib.lib().ns2vc_unet_time_table_floats(sess.h, B)), device="cuda")
        with pytest.raises(_lib.Ns2vcError, match=msg):
            sess.time_table_rows(torch.ones((1, B), device="cuda"), table, rows)
    padded = DenoiserSession(unet, content, prompt, torch.ones((B, S), dtype=torch.bool, device="cuda"))
    with pytest.raises(ValueError, match="ragged"):
        padded.prepare_rows([0])
