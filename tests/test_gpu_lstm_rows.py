"""The LSTM recurrence runs 16 batch rows per CTA from 128 windows up and 8 below.  Rows on either side of a CTA boundary,
and rows of a partial last CTA, give the scores of the same windows run alone (bit for bit, across the two instances),
and batches that end inside a CTA match the oracle."""
import pytest
import torch

from diart_b200 import models, synth

pytestmark = pytest.mark.gpu

SEG_TOL = 1e-4
N = 136     # 16-row instance: eight full CTAs and a partial one of 8 rows


@pytest.fixture(scope="module")
def windows():
    """N consecutive 5 s windows (0.5 s step) of the seeded synthetic stream"""
    stream = synth.synth_audio(80000 + 8000 * (N - 1), seed=4321)
    return torch.from_numpy(synth.windows(stream, N))


@pytest.fixture(scope="module")
def seg_nets(cuda_device, oracle_nets):
    seg_o, _ = oracle_nets
    return seg_o, models.B200PyanNet(seg_o.state_dict()).to(cuda_device)


@pytest.fixture(scope="module")
def oracle33(seg_nets, windows):
    seg_o, _ = seg_nets
    with torch.no_grad():
        return seg_o(windows[:33, None, :])


@pytest.mark.parametrize("B", [1, 15, 16, 17, 33])
def test_segmentation_matches_oracle_at_cta_edges(seg_nets, oracle33, windows, cuda_device, B):
    _, seg_c = seg_nets
    out = seg_c(windows[:B, None, :].to(cuda_device)).cpu()
    assert out.shape == (B, 293, 3)
    err = (out - oracle33[:B]).abs().max().item()
    assert err < SEG_TOL, f"B = {B}: max abs err {err}"


@pytest.fixture(scope="module")
def full(seg_nets, windows, cuda_device):
    _, seg_c = seg_nets
    return seg_c(windows.to(cuda_device)[:, None, :])


def test_wide_batch_matches_oracle(seg_nets, windows, full):
    """the 16-row instance: the windows around the first CTA boundary and the partial last CTA"""
    seg_o, _ = seg_nets
    idx = list(range(14, 19)) + list(range(128, N))
    with torch.no_grad():
        ref = seg_o(windows[idx, None, :])
    err = (full[idx].cpu() - ref).abs().max().item()
    assert err < SEG_TOL, f"max abs err {err}"


def test_rows_across_cta_boundary_are_batch_invariant(seg_nets, windows, full, cuda_device):
    """windows 14-18 straddle the first CTA boundary of both instances"""
    _, seg_c = seg_nets
    x = windows.to(cuda_device)[:, None, :]
    head = seg_c(x[:40])
    five = seg_c(x[14:19])
    assert torch.equal(full[14:19], five)
    assert torch.equal(head[14:19], five)
    for i in range(14, 19):
        assert torch.equal(full[i], seg_c(x[i:i + 1])[0]), f"window {i}"


def test_row_of_partial_last_cta_is_batch_invariant(seg_nets, windows, full, cuda_device):
    """window N - 1 is the last row of a 16-row CTA that holds 8 rows; window 32 of a 33-window batch the only row of
    its 8-row CTA"""
    _, seg_c = seg_nets
    x = windows.to(cuda_device)[:, None, :]
    assert torch.equal(full[N - 1], seg_c(x[N - 1:N])[0])
    assert torch.equal(seg_c(x[:33])[32], seg_c(x[32:33])[0])
