"""Seeded sampler noise (csrc/philox.cuh, ns2vc_b200/noise.py): Philox4x32-10 with counter (t >> 2, c, step, 0) under the
utterance's seed, and Box-Muller of its output pairs.

CPU: the oracle reproduces curand's known-answer vectors and its layout does not depend on T; the seed and argument checks.
GPU: the device generator's raw outputs equal the oracle's bit for bit, its normals lie within 2^-20 * r of the fp64 transform
and look like independent N(0, 1) draws, and the row step kernel's in-register draw equals ``noise.normal_rows`` bit for bit."""
import numpy as np
import pytest
import torch

from ns2vc_b200 import api, noise
from oracle import philox_oracle as po

KAT = [  # (counter, key, output), curand_Philox4x32_10
    ([0, 0, 0, 0], [0, 0], [0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8]),
    ([0xffffffff] * 4, [0xffffffff] * 2, [0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd]),
    ([0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344], [0xa4093822, 0x299f31d0], [0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1]),
]


# ------------------------------------------------------------------------------------------------------------------- CPU
def test_oracle_reproduces_the_known_answer_vectors():
    for ctr, key, want in KAT:
        assert po.philox4x32_10(ctr, key).tolist() == want


def test_layout_does_not_depend_on_T():
    for seed, step in ((0, 0), (12345, 7), ((1 << 63) - 1, po.XT_STEP)):
        a, _ = po.normal(seed, step, 3, 37)
        b, _ = po.normal(seed, step, 3, 1024)
        assert np.array_equal(a, b[:, :37])
    # frame t of channel c is the (t & 3)-th normal of the call (t >> 2, c, step, 0)
    z, _ = po.normal(99, 4, 2, 8)
    o = po.philox4x32_10([1, 1, 4, 0], po.seed_key(99))
    z0, z1, _ = po.box_muller(o[2], o[3])
    assert z[1, 6] == z0 and z[1, 7] == z1


def test_seed_and_argument_checks_raise():
    assert noise.check_seeds([0, (1 << 63) - 1], 2) == [0, (1 << 63) - 1]
    for bad in ([1], [1, -1], [1, 1 << 63]):
        with pytest.raises(ValueError):
            noise.check_seeds(bad, 2)
    x, c, p = torch.zeros(2, 100, 8), torch.zeros(8, 2, 256), torch.zeros(5, 2, 256)
    for kw in (dict(method="ddim", noise_seeds=[1]), dict(method="ddim", noise_seeds=[1, -2]),
               dict(method="ddpm", noise_seeds=[1, 1 << 63]), dict(method="ddim", noise_seeds=[1, 2], noise=torch.zeros(1)),
               dict(method="ddim", noise_seeds=[1, 2], eta=1.5), dict(method="ddim", noise_seeds=[1, 2], eta=-0.1),
               dict(method="unipc", noise_seeds=[1, 2])):
        with pytest.raises(ValueError):
            api.sample_latents(None, x, c, p, None, **kw)
    items = [(torch.zeros(100, 4), torch.zeros(4, 256), torch.zeros(3, 256))] * 3
    with pytest.raises(ValueError):
        api.sample_utterances(None, items, method="ddim", noise_seeds=[1, 2])


# ------------------------------------------------------------------------------------------------------------------- GPU
def _device_philox(ctr: np.ndarray, key: np.ndarray):
    from ns2vc_b200 import _lib
    n = ctr.shape[0]
    c = torch.from_numpy(ctr.astype(np.int64)).to(torch.int32).cuda()       # (uint32 bits carried in int32)
    k = torch.from_numpy(key.astype(np.int64)).to(torch.int32).cuda()
    raw = torch.empty((n, 4), dtype=torch.int32, device="cuda")
    z = torch.empty((n, 4), dtype=torch.float32, device="cuda")
    _lib.check(_lib.lib().ns2vc_check_philox(c.data_ptr(), k.data_ptr(), n, raw.data_ptr(), z.data_ptr(), None))
    torch.cuda.synchronize()
    return raw.cpu().numpy().view(np.uint32), z.cpu().double().numpy()


def _random_cases(n, seed):
    rng = np.random.default_rng(seed)
    ctr = rng.integers(0, 1 << 32, size=(n, 4), dtype=np.uint64).astype(np.uint32)
    key = rng.integers(0, 1 << 32, size=(n, 2), dtype=np.uint64).astype(np.uint32)
    ctr[:len(KAT)] = [k[0] for k in KAT]
    key[:len(KAT)] = [k[1] for k in KAT]
    return ctr, key


@pytest.mark.gpu
def test_device_generator_matches_the_oracle_bit_for_bit():
    ctr, key = _random_cases(1 << 16, 1)
    raw, _ = _device_philox(ctr, key)
    assert np.array_equal(raw, po.philox4x32_10(ctr, key))
    assert raw[:len(KAT)].tolist() == [k[2] for k in KAT]


@pytest.mark.gpu
def test_device_normals_are_within_2e20_radius_of_fp64():
    ctr, key = _random_cases(1 << 18, 2)
    raw, z = _device_philox(ctr, key)
    for pair in (0, 1):
        z0, z1, r = po.box_muller(raw[:, 2 * pair], raw[:, 2 * pair + 1])
        for got, want in ((z[:, 2 * pair], z0), (z[:, 2 * pair + 1], z1)):
            err = np.abs(got - want)
            assert (err <= 2.0 ** -20 * r).all(), f"worst err / r = {(err / r).max():.3e}"


@pytest.mark.gpu
def test_normal_rows_look_like_independent_standard_normals():
    from scipy import stats
    seeds = [0, 1, 2, (1 << 63) - 1]
    a = noise.normal_rows(seeds, 100, T=2560, step=0).double()             # 1 024 000 draws
    v = a.flatten().cpu().numpy()
    n = v.size
    assert abs(v.mean()) < 5 / np.sqrt(n) and abs(v.var() - 1) < 5 * np.sqrt(2 / n)
    assert abs(stats.skew(v)) < 5 * np.sqrt(6 / n) and abs(stats.kurtosis(v)) < 5 * np.sqrt(24 / n)
    assert stats.kstest(v, "norm").pvalue > 1e-4
    lim = 5 / np.sqrt(a[0].numel())

    def corr(x, y):
        return float(torch.corrcoef(torch.stack([x.flatten(), y.flatten()]))[0, 1])
    assert abs(corr(a[0], a[1])) < lim and abs(corr(a[1], a[3])) < lim                       # across seeds
    b = noise.normal_rows(seeds, 100, T=2560, step=1).double()
    assert abs(corr(a[0], b[0])) < lim                                                      # across steps
    assert abs(corr(a[2, :50], a[2, 50:])) < 5 / np.sqrt(a[2, :50].numel())                   # across channels
    assert abs(corr(a[2, :, :-1], a[2, :, 1:])) < lim                                       # neighbouring frames
    # the device fill equals the oracle's normals to 2^-20 r, zeros past each length
    got = noise.normal_rows([7, 8], 5, lengths=[37, 64], step=3).double().cpu().numpy()
    for j, (s, t) in enumerate(((7, 37), (8, 64))):
        want, r = po.normal(s, 3, 5, t)
        assert (np.abs(got[j, :, :t] - want) <= 2.0 ** -20 * r).all()
        assert not got[j, :, t:].any()


@pytest.mark.gpu
def test_row_kernel_draw_equals_normal_rows_bit_for_bit():
    """DDIM rows with x = x0 = 0 and unit coefficients give x_new = 0 + 1 * noise, DDPM rows likewise: the noise itself."""
    from ns2vc_b200 import _lib
    L = _lib.lib()
    B, C, T = 4, 5, 37
    seeds = [3, 1 << 40, 3, (1 << 63) - 1]
    steps = [0, 17, 999, -1]                                  # row 3 is empty
    methods = [_lib.ROW_DDIM, _lib.ROW_DDPM, _lib.ROW_DDIM, _lib.ROW_DDPM]
    ddim = (_lib.DdimCoef * 1000)(*[_lib.DdimCoef(1.0, 1.0, 1.0, 1.0, 1.0, 0)] * 1000)
    ddpm = (_lib.DdpmCoef * 1000)(*[_lib.DdpmCoef(0.0, 0.0, 1.0, 1)] * 1000)
    dev = lambda arr: torch.frombuffer(bytearray(bytes(arr)), dtype=torch.uint8).cuda()
    ddim_d, ddpm_d = dev(ddim), dev(ddpm)
    i32 = lambda v: torch.tensor(v, dtype=torch.int32, device="cuda")
    sd = torch.tensor(seeds, dtype=torch.int64, device="cuda")
    meth, base, k = i32(methods), i32([0] * B), i32(steps)
    x = torch.zeros((B, C, T), device="cuda")
    x0 = torch.zeros_like(x)
    out = torch.full_like(x, float("nan"))
    flags = torch.zeros(B, dtype=torch.int32, device="cuda")
    _lib.check(L.ns2vc_sampler_step_rows_seeded(x.data_ptr(), x0.data_ptr(), None, None, None, None, None, ddpm_d.data_ptr(),
                                                ddim_d.data_ptr(), sd.data_ptr(), T, meth.data_ptr(), base.data_ptr(), k.data_ptr(), None,
                                                None, out.data_ptr(), C * T, B, flags.data_ptr(), None))
    torch.cuda.synchronize()
    for b in range(3):
        want = noise.normal_rows([seeds[b]], C, T=T, step=steps[b])[0]
        assert torch.equal(out[b], want), b
    assert not out[3].any()
    assert k.tolist() == [1, 18, 1000, -1] and not flags.any()
    # in place (x_new = x_in) and the NaN flag of the row that holds one
    x[2, 1, 5] = float("nan")
    _lib.check(L.ns2vc_sampler_step_rows_seeded(x.data_ptr(), x0.data_ptr(), None, None, None, None, None, ddpm_d.data_ptr(),
                                                ddim_d.data_ptr(), sd.data_ptr(), T, meth.data_ptr(), base.data_ptr(), k.data_ptr(), None,
                                                None, x.data_ptr(), C * T, B, flags.data_ptr(), None))
    torch.cuda.synchronize()
    assert flags.tolist() == [0, 0, 1, 0]
    assert torch.equal(x[0], noise.normal_rows([seeds[0]], C, T=T, step=1)[0])
    # a row of length T_b = 37 reads the same noise as a longer one at t < 37
    long = noise.normal_rows([seeds[1]], C, T=1024, step=17)[0]
    assert torch.equal(out[1], long[:, :T])
