"""Host side of the stage-by-stage tests of the default networks (tests/test_gpu_net_stages.py): the stage hooks refuse bad
arguments without touching a device, the sinc filter table the library builds is the oracle's, and the layered float64
evaluation the GPU tests compare against is the float64 forward."""
import ctypes as C

import numpy as np
import torch

from diart_b200 import _lib, synth
from oracle import nets


def test_stage_hooks_refuse_bad_arguments_without_gpu():
    lib = _lib.lib()
    out = np.zeros(16, np.float32)
    dims = (C.c_int * 4)()
    fake = C.create_string_buffer(4096)          # stands for a handle and a device pointer: a refusal reads neither
    p = C.addressof(fake)
    launches = lib.dg_launch_count()
    assert lib.dg_seg_debug_stage(None, p, 1, 80000, 0, 0, out.ctypes.data, out.size, dims) == -1
    assert b"dg_seg_debug_stage" in lib.dg_last_error()
    assert lib.dg_emb_debug_stage(None, p, None, 1, 80000, 0, 0, 0, 0, out.ctypes.data, out.size, dims) == -1
    assert b"dg_emb_debug_stage" in lib.dg_last_error()
    for stage in (-1, 11):
        assert lib.dg_seg_debug_stage(p, p, 1, 80000, 0, stage, out.ctypes.data, out.size, dims) == -1
    for stage in (-1, 13):
        assert lib.dg_emb_debug_stage(p, p, p, 1, 80000, 293, 3, 0, stage, out.ctypes.data, out.size, dims) == -1
    assert lib.dg_emb_debug_stage(p, p, None, 1, 80000, 293, 3, 0, 9, out.ctypes.data, out.size, dims) == -1   # pooling needs weights
    assert lib.dg_seg_debug_stage(p, p, 0, 80000, 0, 0, out.ctypes.data, out.size, dims) == -1
    assert lib.dg_seg_debug_stage(p, p, 1, 80000, -8000, 0, out.ctypes.data, out.size, dims) == -1
    assert lib.dg_launch_count() == launches


def _library_filters(fb):
    lo = np.ascontiguousarray(fb.low_hz_.detach().numpy().reshape(40), np.float32)
    bd = np.ascontiguousarray(fb.band_hz_.detach().numpy().reshape(40), np.float32)
    got = np.empty((251, 80), np.float32)
    assert _lib.lib().dg_selftest_sinc_filters_host(lo.ctypes.data, bd.ctypes.data, got.ctypes.data) == 0
    return got.T                                  # [filter][tap]


def test_sinc_filter_table_is_the_oracles():
    """The library builds ParamSincFB.filters() in float32 with libm's sinf / cosf, torch with its own vectorised ones.  94 % of
    the taps are bit-equal; the rest differ by at most 1.3e-6 of their filter's largest tap (measured; the differences of two
    nearby sines or cosines of the narrow low bands amplify the last bit).  Both tables are 4.2e-6 of a filter's RMS from the
    float64 evaluation, so neither is the better one.  Filters at the `low_hz` floor and the `high` clamp included."""
    for seg in (nets.make_segmentation(), nets.make_embedding()):
        fb = seg.sincnet.conv1d[0].filterbank
        with torch.no_grad():
            fb.low_hz_[0] = 0.0                    # low = min_low_hz exactly
            fb.band_hz_[39] = 9000.0               # high clamps to sample_rate / 2
            want32 = fb.filters()[:, 0, :].numpy()
            import copy
            want64 = copy.deepcopy(fb).double().filters()[:, 0, :].numpy()
        got = _library_filters(fb)
        assert np.isfinite(got).all()
        peak = np.abs(want32).max(axis=1, keepdims=True)
        ulp = np.abs(got - want32) / peak
        rel64 = np.abs(got - want64).max(axis=1) / np.sqrt((want64 ** 2).mean(axis=1))
        print(f"filters: max |lib - torch32| / peak {ulp.max():.2e}, bit-equal taps {np.mean(got == want32):.3f}, "
              f"max |lib - float64| / rms {rel64.max():.2e}")
        assert np.mean(got == want32) > 0.9 and ulp.max() < 2.5e-6
        assert rel64.max() < 1e-5


def test_layered_float64_evaluation_is_the_float64_forward():
    x = torch.from_numpy(synth.windows(synth.synth_audio(16000 + 8000, seed=5), 2, chunk=16000))[:, None, :].double()
    seg = nets.float64_copy(nets.make_segmentation())
    st = nets.segmentation_stages(seg, x)
    taps = {}
    with torch.no_grad():
        want = torch.nn.Module.__call__(seg, x, taps)
    assert st["scores"].dtype == torch.float64 and torch.equal(st["scores"], want)
    assert torch.equal(st["sinc_norm2"], taps["sincnet"]) and torch.equal(st["lstm3"], taps["lstm"])
    emb = nets.float64_copy(nets.make_embedding())
    w = torch.rand((2, 53, 3), generator=torch.Generator().manual_seed(1), dtype=torch.float64)
    se = nets.embedding_stages(emb, x, w)
    taps = {}
    with torch.no_grad():
        trunk = emb.trunk(x, taps)
        want = torch.stack([emb.embedding(emb.stats_pool(trunk, w[:, :, k])) for k in range(3)], dim=1)
    assert torch.allclose(se["embedding"], want, rtol=0, atol=1e-13)      # one Linear over (B, K, 3000) instead of K over (B, 3000)
    for i in range(5):
        assert torch.equal(se[f"tdnn{i}"], taps[f"tdnn{i}"].transpose(1, 2))
    # the statistics the front end normalises the waveform with
    y = (x - st["wmean"][:, None, None]) * st["wrstd"][:, None, None] * seg.sincnet.wav_norm1d.weight + seg.sincnet.wav_norm1d.bias
    assert torch.allclose(y, seg.sincnet.wav_norm1d(x), rtol=0, atol=1e-12)
    # the copy convolves with the float32 filters, cast up
    f32 = nets.make_segmentation().sincnet.conv1d[0].filterbank.filters().detach()
    assert torch.equal(seg.sincnet.conv1d[0].filterbank.filters(), f32.double())
