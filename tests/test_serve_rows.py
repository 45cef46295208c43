"""Row-scoped admission in ``serve.ConversionServer``: requests admitted while other slots sit at mid-run steps.

An admission re-prepares only the newcomers' rows and the rows of slots freed since the last admission.  The arrival script
below admits one request beside residents at steps 1 to 7, one into a slot freed two ticks earlier, and one while two other
freed slots go back to blank rows.  Each result must equal, bit for bit, the same script served with every admission
re-preparing every slot, and match ``convert_batch`` of the request alone as ``test_serve.py`` checks it."""
import pytest
import torch

from ns2vc_b200 import serve
from test_convert import SR
from test_serve import MAX_FRAMES, MAX_PROMPT, SLOTS, STEPS, _alone, _check_parity, chain  # noqa: F401  (chain: the shared fixture)

ARRIVALS = {0: [0], 1: [1], 3: [2], 5: [3], 6: [4], 13: [5]}   # tick -> requests submitted just before it


def _serve(models, wavs, prompt, xs, method, full):
    srv = serve.ConversionServer(*models, slots=SLOTS, max_frames=MAX_FRAMES, max_prompt_frames=MAX_PROMPT, method=method, steps=STEPS)
    rows_seen = []
    if full:
        srv._prepare_rows = lambda rows: (rows_seen.append(list(rows)), srv._prepare_all())
    else:
        inner = srv._prepare_rows
        srv._prepare_rows = lambda rows: (rows_seen.append(list(rows)), inner(rows))
    req, res, lat = {}, {}, {}
    while len(res) < len(wavs):
        for i in ARRIVALS.get(srv.ticks, ()):
            req[srv.submit(wavs[i], SR, prompt, x_T=xs[i])] = i
        assert not srv.table.idle, "the script leaves the server idle before every request is served"
        done = srv.tick()
        res.update({req[tk]: v for tk, v in done.items()})
        lat.update({req[tk]: v for tk, v in srv.last_latents.items()})
    assert srv.table.idle
    return res, lat, rows_seen


@pytest.mark.gpu
@pytest.mark.parametrize("method", ["unipc", "dpmsolver"])
def test_admissions_beside_mid_run_slots(chain, method):  # noqa: F811
    models, wavs, prompt, xs = chain
    res, lat, rows = _serve(models, wavs, prompt, xs, method, full=False)
    # tick 0 prepares every slot (the first prepare); then request 1 alone, 2 and 3 alone, 4 into the slot request 0 freed,
    # and 5 into slot 1 while slots 2 and 3, freed since the last admission, go back to blank rows
    assert rows == [[1], [2], [3], [0], [1, 2, 3]], rows
    ref, ref_lat, _ = _serve(models, wavs, prompt, xs, method, full=True)
    for i in range(len(wavs)):
        assert torch.equal(lat[i], ref_lat[i]), f"{method} request {i}: latent differs from the full-prepare server"
        assert torch.equal(res[i], ref[i]), f"{method} request {i}: audio differs from the full-prepare server"
    _check_parity(models, wavs, prompt, xs, method, res, lat)
    for i in range(len(wavs)):
        la, aa = _alone(models, wavs, prompt, xs, method, i)
        assert torch.equal(lat[i], la) and torch.equal(res[i], aa), f"{method} request {i}: not bit-identical to its conversion alone"
