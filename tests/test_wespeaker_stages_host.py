"""Host side of the stage-by-stage tests of variant B (WeSpeaker ResNet34, tests/test_zz_wespeaker_stages.py) and of powerset
segmentation: the layered float64 evaluation the GPU tests compare against is the float64 forward, the kaldi fbank tables the
library builds are the oracle's, and the hooks refuse bad arguments without touching a device."""
import ctypes as C

import numpy as np
import torch

from diart_b200 import _lib, synth
from oracle import fbank_linear, nets


def test_layered_float64_evaluation_is_the_float64_forward():
    torch.set_num_threads(8)
    x = torch.from_numpy(synth.windows(synth.synth_audio(16000 + 8000, seed=5), 2, chunk=16000))[:, None, :].double()
    net = nets.float64_copy(nets.make_wespeaker())
    assert next(net.parameters()).dtype == torch.float64
    w = torch.rand((2, 53, 3), generator=torch.Generator().manual_seed(1), dtype=torch.float64)
    st = nets.wespeaker_stages(net, x, w)
    with torch.no_grad():
        fb = net.compute_fbank(x)
        maps = net.resnet.maps(fb)
        dedup = torch.nn.Module.__call__(net, x, w[:, :, 1])           # one speaker through forward
        rows = net.forward_dedup(x, w)
    assert st["logmel"].dtype == torch.float64 and st["logmel"].shape == (2, 98, 80)
    assert torch.equal(st["logmel"] - st["logmel"].mean(dim=1, keepdim=True), fb)
    assert torch.equal(st["block15"], maps.permute(0, 3, 2, 1))         # (U, C, mel, time) -> (U, time, mel, C)
    assert st["stem"].shape == (2, 98, 80, 32) and st["block3"].shape == (2, 49, 40, 64)
    assert st["block7"].shape == (2, 25, 20, 128) and st["block15"].shape == (2, 13, 10, 256)
    assert torch.equal(st["embedding"], rows)
    assert torch.equal(st["embedding"][:, 1], dedup)


def test_powerset_layered_evaluation_is_the_forward():
    x = torch.from_numpy(synth.windows(synth.synth_audio(16000 + 8000, seed=5), 2, chunk=16000))[:, None, :].double()
    net = nets.float64_copy(nets.make_powerset_segmentation())
    st = nets.segmentation_stages(net, x)
    taps = {}
    with torch.no_grad():
        want = torch.nn.Module.__call__(net, x, taps)
    assert torch.equal(st["log_probabilities"], taps["log_probabilities"])
    assert torch.equal(st["scores"], want) and st["scores"].shape == (2, want.shape[1], 3)
    assert torch.equal(st["lstm3"], taps["lstm"])


def test_fbank_tables_are_the_oracles():
    """The library builds the [514, 400] frame operator and the [80, 257] mel banks in double and rounds them once to float32.
    The banks are then oracle.fbank_linear's rounded to nearest (measured: all bit-equal).  The operator sums its products in
    another order than numpy: 99.8 % of the entries are bit-equal and the rest lie within one float32 ulp of the operator's
    largest entry (measured 0.50 of it) -- entries near zero have no relative bound.  torchaudio builds its banks in float32
    arithmetic; they are 1.4e-5 away from these in absolute terms (weights <= 1), printed here and left to the log-mel bar."""
    op = np.empty((514, 400), np.float32)
    banks = np.empty((80, 257), np.float32)
    assert _lib.lib().dg_selftest_fbank_tables_host(op.ctypes.data, banks.ctypes.data) == 0
    want_op, want_banks = fbank_linear.frame_operator(), fbank_linear.mel_banks()
    ulp_max = np.spacing(np.float32(np.abs(want_op).max()))
    err = np.abs(op.astype(np.float64) - want_op).max()
    print(f"operator: bit-equal {np.mean(op == want_op.astype(np.float32)):.4f}, max |lib - f64| {err / ulp_max:.2f} ulp of its largest entry")
    assert np.mean(op == want_op.astype(np.float32)) > 0.99
    assert err <= ulp_max
    assert np.array_equal(banks, want_banks.astype(np.float32))
    from torchaudio.compliance.kaldi import get_mel_banks

    tb = np.pad(get_mel_banks(80, 512, 16000.0, 20.0, 0.0, 100.0, -500.0, 1.0)[0].numpy(), ((0, 0), (0, 1)))
    print(f"banks: torchaudio float32 vs library, max abs {np.abs(tb - banks).max():.2e}")
    assert np.abs(tb - banks).max() < 5e-5


def test_hooks_refuse_bad_arguments_without_gpu():
    lib = _lib.lib()
    launches = lib.dg_launch_count()
    out = np.zeros(16, np.float32)
    assert lib.dg_selftest_fbank_tables_host(None, out.ctypes.data) == -1
    assert lib.dg_selftest_fbank_tables_host(out.ctypes.data, None) == -1
    assert b"dg_selftest_fbank_tables_host" in lib.dg_last_error()
    dims = (C.c_int * 4)()
    fake = C.create_string_buffer(4096)
    p = C.addressof(fake)
    for stage in (-1, 11):                        # the powerset stages are 0..10 like the multilabel ones
        assert lib.dg_seg_debug_stage(p, p, 1, 80000, 0, stage, out.ctypes.data, out.size, dims) == -1
        assert b"dg_seg_debug_stage" in lib.dg_last_error()
    assert lib.dg_emb_debug_trunk(None, p, 1, 80000, -2, out.ctypes.data, out.size, dims) == -1
    assert b"dg_emb_debug_trunk" in lib.dg_last_error()
    assert lib.dg_launch_count() == launches
