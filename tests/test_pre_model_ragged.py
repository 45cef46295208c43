"""Ragged condition encoders: ``Pre_model.infer(per_utterance=True)`` (C-ABI ``ns2vc_pre_infer_ragged``).

Contract: row b equals ``Pre_model.infer`` of c[b, :, :T_b], refer[b, :, :S_b] alone; frames past T_b / S_b are exactly 0 and
input values there are never read.  Each row is judged against the fp64 oracle of that utterance alone with the rule of
``test_numerics_fp64.test_condition_encoders_vs_fp64`` (|gpu - ref| <= max(1e-3 |ref| + 1e-4 rms, 2 max(e32, e_qk)), e_qk the
oracle's own change when only the scores are formed from bf16 hi/lo pairs), and against its own B = 1 GPU run.  The padded
program is run on the same inputs to show that the rule tells the two programs apart."""
import math

import pytest
import torch

from oracle import pre_model_oracle as po
from test_numerics_fp64 import (PRE_B, PRE_FULL, PRE_LENGTHS, PRE_REFER_LENGTHS, PRE_S, PRE_T, TARGET_SCORE_STD, ScoreStd,
                                _pre_scores, _self_attention_3xbf16_scores, contract, pre_inputs)

pytestmark = pytest.mark.gpu
RTOL, ATOL = 1e-3, 1e-4
_models = {}


def regime_state_dict(regime):
    """The weights of test_condition_encoders_vs_fp64: seed-1 synthetic init, or with every self-attention's q and k scaled so
    that the fp64 score std is ~4 ("sharp")."""
    from ns2vc_b200.pre_model import Pre_model
    shapes = {k: tuple(v.shape) for k, v in Pre_model(PRE_FULL).state_dict().items()}
    sd = po.synth_state_dict(shapes, seed=1)
    if regime == "sharp":
        c, refer, lengths, refer_lengths = pre_inputs()
        with ScoreStd(po, "self_attention", _pre_scores) as rec, torch.no_grad():
            po.pre_model_infer({k: v.double() for k, v in sd.items()}, c.double(), refer.double(), lengths, refer_lengths, 6, 6)
        g = math.sqrt(TARGET_SCORE_STD / (sum(rec.std.values()) / len(rec.std)))
        for k in sd:
            if k.endswith("self_attn.in_proj_weight"):
                C = sd[k].shape[1]
                sd[k] = torch.cat([sd[k][:2 * C] * g, sd[k][2 * C:]])
    return sd


def model(regime):
    if regime not in _models:
        from ns2vc_b200.pre_model import Pre_model
        sd = regime_state_dict(regime)
        m = Pre_model(PRE_FULL)
        m.load_state_dict(sd, strict=True)
        _models[regime] = (m.to("cuda").eval(), sd)
    return _models[regime]


def data(c, refer, lengths=PRE_LENGTHS, refer_lengths=PRE_REFER_LENGTHS):
    return (c.cuda(), refer.cuda(), None, None, None, torch.tensor(lengths), torch.tensor(refer_lengths), None)


def run(m, c, refer, per_utterance=True, lengths=PRE_LENGTHS, refer_lengths=PRE_REFER_LENGTHS):
    content, prompt = m.infer(data(c, refer, lengths, refer_lengths), per_utterance=per_utterance)
    torch.cuda.synchronize()
    return content.cpu(), prompt.cpu()


def alone_oracle(sd, c, refer, b, dtype):
    Tb, Sb = PRE_LENGTHS[b], PRE_REFER_LENGTHS[b]
    with torch.no_grad():
        return po.pre_model_infer({k: v.to(dtype) for k, v in sd.items()}, c[b:b + 1, :, :Tb].to(dtype), refer[b:b + 1, :, :Sb].to(dtype),
                                  torch.tensor([Tb]), torch.tensor([Sb]), 6, 6)


def row_ratios(sd, c, refer, content, prompt):
    """Worst elementwise err/tol of each row's content and prompt against the fp64 oracle of the row alone.  As in
    test_condition_encoders_vs_fp64, the floor of an output is the largest over the batch of the oracle's fp32 error and its
    3xBF16-score change."""
    rows = []
    for b in range(PRE_B):
        Tb, Sb = PRE_LENGTHS[b], PRE_REFER_LENGTHS[b]
        ref_c, ref_p = alone_oracle(sd, c, refer, b, torch.float64)
        r32_c, r32_p = alone_oracle(sd, c, refer, b, torch.float32)
        orig = po.self_attention
        po.self_attention = _self_attention_3xbf16_scores
        try:
            qk_c, qk_p = alone_oracle(sd, c, refer, b, torch.float64)
        finally:
            po.self_attention = orig
        rows.append([(got, ref, max((r32.double() - ref).abs().max().item(), (rqk - ref).abs().max().item()))
                     for got, ref, r32, rqk in ((content[:Tb, b:b + 1], ref_c, r32_c, qk_c), (prompt[:Sb, b:b + 1], ref_p, r32_p, qk_p))])
    floors = [max(r[k][2] for r in rows) for k in range(2)]
    return [tuple(contract(got, ref, floors[k], ref)[0] for k, (got, ref, _) in enumerate(r)) for r in rows]


@pytest.mark.parametrize("regime", ["synthetic", "sharp"])
def test_ragged_rows_match_each_utterance_alone_vs_fp64(regime):
    m, sd = model(regime)
    c, refer, _, _ = pre_inputs()
    content, prompt = run(m, c, refer)
    ratios = row_ratios(sd, c, refer, content, prompt)
    print(f"\n== ragged encoders {regime}: B={PRE_B} T={PRE_T} S={PRE_S}")
    bad = []
    for b, (rc, rp) in enumerate(ratios):
        print(f"   row {b} (T_b={PRE_LENGTHS[b]:3d}, S_b={PRE_REFER_LENGTHS[b]:3d}): content err/tol {rc:.3f}  prompt err/tol {rp:.3f}")
        if rc > 1.0 or rp > 1.0:
            bad.append(f"row {b} (T_b={PRE_LENGTHS[b]}, S_b={PRE_REFER_LENGTHS[b]}): content {rc:.3f}, prompt {rp:.3f}")
    assert not bad, f"ragged encoders {regime} vs the fp64 oracle of each utterance alone:\n" + "\n".join(bad)


def _close(a, b):
    err = (a.double() - b.double()).abs()
    return bool((err <= ATOL + RTOL * b.double().abs()).all()), err.max().item()


def test_ragged_rows_match_their_own_b1_runs():
    m, _ = model("synthetic")
    c, refer, _, _ = pre_inputs()
    content, prompt = run(m, c, refer)
    bad, bitwise = [], []
    for b in range(PRE_B):
        Tb, Sb = PRE_LENGTHS[b], PRE_REFER_LENGTHS[b]
        oc, op = run(m, c[b:b + 1, :, :Tb].contiguous(), refer[b:b + 1, :, :Sb].contiguous(), per_utterance=False, lengths=(Tb,),
                     refer_lengths=(Sb,))
        for name, got, own in (("content", content[:Tb, b:b + 1], oc), ("prompt", prompt[:Sb, b:b + 1], op)):
            ok, mx = _close(got, own)
            if not ok:
                bad.append(f"row {b} (T_b={Tb}, S_b={Sb}) {name}: max|diff| {mx:.3e}")
        bitwise.append(torch.equal(content[:Tb, b:b + 1], oc) and torch.equal(prompt[:Sb, b:b + 1], op))
    print(f"\nragged encoder rows bit-identical to their B=1 runs: {bitwise}")
    assert not bad, "\n".join(bad)


def test_exact_zeros_garbage_inputs_and_poisoned_workspace():
    m, _ = model("synthetic")
    c, refer, _, _ = pre_inputs()
    content, prompt = run(m, c, refer)
    for b in range(PRE_B):
        assert not content[PRE_LENGTHS[b]:, b].any(), f"content row {b}: frames past T_b={PRE_LENGTHS[b]} are not exactly 0"
        assert not prompt[PRE_REFER_LENGTHS[b]:, b].any(), f"prompt row {b}: frames past S_b={PRE_REFER_LENGTHS[b]} are not exactly 0"
    cg, rg = c.clone(), refer.clone()
    for b in range(PRE_B):
        cg[b, :, PRE_LENGTHS[b]:] = float("nan") if b % 2 else 1e30
        rg[b, :, PRE_REFER_LENGTHS[b]:] = 1e30 if b % 2 else float("nan")
    dc, dp = run(m, cg, rg)
    for b in range(PRE_B):
        assert torch.equal(dc[:, b], content[:, b]) and torch.equal(dp[:, b], prompt[:, b]), f"row {b}: NaN / 1e30 padding changed the result"
    ws = m.workspace(PRE_B, PRE_T, PRE_S, torch.device("cuda", torch.cuda.current_device()))
    ws.fill_(0xFF)
    pc, pp = run(m, c, refer)
    ws.zero_()
    zc, zp = run(m, c, refer)
    assert torch.equal(pc, zc) and torch.equal(pp, zp), "a 0xFF-filled workspace changed the ragged result"
    assert torch.equal(zc, content) and torch.equal(zp, prompt)


def test_padded_and_ragged_programs_alternate_on_one_workspace():
    m, _ = model("synthetic")
    c, refer, _, _ = pre_inputs()
    first = {True: run(m, c, refer, True), False: run(m, c, refer, False)}
    counts = {}
    for k, ragged in enumerate((True, False, True, False, False, True)):
        got = run(m, c, refer, ragged)
        counts[ragged] = m.launch_count()
        name = "ragged" if ragged else "padded"
        assert torch.equal(got[0], first[ragged][0]) and torch.equal(got[1], first[ragged][1]), f"call {k} ({name}) differs from its program's first result"
    assert not torch.equal(first[True][0], first[False][0])
    print(f"\nlaunches per infer: padded {counts[False]}, ragged {counts[True]}")
    assert counts[True] == counts[False]


def test_padded_program_misses_the_lone_utterance_oracle():
    """The gap the ragged program closes: under the same rule the padded program's short rows miss the oracle of the utterance
    alone (the conv-FFN reads LN2's beta past T_b, ref_enc pools over all S prompt frames)."""
    m, sd = model("synthetic")
    c, refer, _, _ = pre_inputs()
    content, prompt = run(m, c, refer, per_utterance=False)
    ratios = row_ratios(sd, c, refer, content, prompt)
    for b, (rc, rp) in enumerate(ratios):
        print(f"   padded row {b} (T_b={PRE_LENGTHS[b]:3d}, S_b={PRE_REFER_LENGTHS[b]:3d}): content err/tol {rc:.1f}  prompt err/tol {rp:.1f}")
    short = [b for b in range(PRE_B) if PRE_LENGTHS[b] < PRE_T]
    assert all(ratios[b][0] > 1.0 for b in short), "the padded program met the lone-utterance rule on a short row"
