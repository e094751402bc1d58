"""CPU: the oracle restatement against the unmodified reference, stage by stage with amplified inputs (end-to-end
parity alone is blind to e.g. a wrong GELU variant in corr_mlp, SURVEY Appendix A).  The reference's outputs on these
seeded inputs are pinned in tests/golden/reference_stages.npz (oracle/make_reference_stages.py)."""
import pytest
import torch

from cases import O, reference_golden, stage_inputs
from cotracker_b200.synthetic import seeded_state_dict


@pytest.fixture(scope="module")
def ref():
    sd = seeded_state_dict(2024, offline=True, window_len=60, head_gain=10.0, vis_gain=100.0)
    return stage_inputs(), sd


def _max_err(got, key):
    idx, want = reference_golden("reference_stages", key)
    got = got.reshape(-1)
    if idx is not None:
        got = got[idx]
    return float((got.double() - want.double()).abs().max()), float(want.abs().max())


def test_updateformer_amplified(ref):
    x, sd = ref
    with torch.no_grad():
        got = O.updateformer(sd, x["uf_x"])
    err, scale = _max_err(got, "updateformer")
    assert err < 1e-4 * max(1.0, scale)


def test_corr_volume_and_corr_mlp_amplified(ref):
    x, sd = ref
    with torch.no_grad():
        got = O.correlation_volume(x["corr_fm"][0], x["corr_sup"][0], x["corr_coords"])
        assert _max_err(got, "corr_volume")[0] < 1e-4
        # the reference's own volume x10 (out of the regime where erf == tanh GELU) into both MLPs
        big = reference_golden("reference_stages", "corr_volume")[1].reshape(got.shape) * 10
        assert _max_err(O.mlp(sd, "corr_mlp", big, "none"), "corr_mlp_big")[0] < 1e-4
        assert _max_err(O.mlp(sd, "corr_mlp", big, "tanh"), "corr_mlp_big")[0] > 1e-4


def test_support_features(ref):
    x, sd = ref
    with torch.no_grad():
        got = O.support_features(x["sup_fm"][0], x["sup_qf"][0], x["sup_qc"][0])
    assert _max_err(got, "support")[0] < 1e-5


def test_posenc_and_time_embedding(ref):
    x, sd = ref
    assert torch.equal(O.posenc(x["posenc_x"]), reference_golden("reference_stages", "posenc")[1])
    for t in (60, 16, 7):
        assert torch.allclose(O.time_embedding(sd, t), reference_golden("reference_stages", f"time_embed_{t}")[1], atol=0)


def test_encoder_and_pyramid(ref):
    x, sd = ref
    with torch.no_grad():
        assert _max_err(O.encoder(sd, x["enc_v"]), "fnet")[0] < 1e-4


def test_offline_forward_live(ref):
    x, sd = ref
    with torch.no_grad():
        gc, gv, gq = O.offline_forward(sd, x["fwd_video"], x["fwd_q"], iters=3)
    wc = reference_golden("reference_stages", "fwd_coords")[1]
    wv = reference_golden("reference_stages", "fwd_vis")[1]
    assert float((gc - wc).abs().max()) < 1e-4 and float((gv - wv).abs().max()) < 1e-5
    assert float((wc[0, -1] - wc[0, 0]).abs().max()) > 0.5   # tracks move
