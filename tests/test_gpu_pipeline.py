"""End-to-end parity of the fused pipeline step (dg_pipeline_step) and of the SpeakerDiarization drop-in
against the oracle pipeline (reference diarization.py:177-203 restated in oracle/pipeline.py).

Bars: segmentation scores within 1e-4, unit-norm embeddings within 1e-4 (float32 re-association only),
speaker maps IDENTICAL to what the oracle clustering produces from the same scores/embeddings, and
identical to the oracle's own end-to-end maps unless the oracle's decision margin at the first differing
chunk is below the float tolerance (reported, never silently skipped)."""
import numpy as np
import pytest
import torch

from diart_b200 import _lib, blocks, models, synth
from diart_b200.blocks.utils import Binarize
from diart_b200.core import SlidingWindow, SlidingWindowFeature
from oracle.clustering import OracleClustering
from oracle.pipeline import OraclePipeline

pytestmark = pytest.mark.gpu
N_CHUNKS, BATCH = 48, 16


@pytest.fixture(scope="module")
def stream():
    return synth.synth_audio(80000 + 8000 * (N_CHUNKS - 1), seed=4242, num_speakers=4)


def make_pipeline(oracle_nets, device, **kw):
    seg_o, emb_o = oracle_nets
    config = blocks.SpeakerDiarizationConfig(
        segmentation=models.SegmentationModel(models.B200SegmentationLoader(seg_o.state_dict())),
        embedding=models.EmbeddingModel(models.B200EmbeddingLoader(emb_o.state_dict())), device=device, **kw)
    return blocks.SpeakerDiarization(config)


def window_form(pipe, num_samples=80000):
    """withdraw the hop hint: the sinc layer then runs once per window instead of once over the stream's unique samples"""
    h = pipe._ensure_fused(num_samples)[0]
    _lib.check(_lib.lib().dg_pipeline_set_hop(h, 0))
    return pipe


@pytest.mark.parametrize("sinc_form", ["stream", "window"])
@pytest.mark.parametrize("params", [dict(), dict(tau_active=0.5, rho_update=0.2, delta_new=0.8, max_speakers=4)])
def test_fused_step_matches_oracle(params, sinc_form, oracle_nets, stream, cuda_device):
    """the batches are consecutive windows of one stream: with the hop hint (default) the sinc layer takes the stream
    form, without it the per-window form; both must meet the same bars"""
    pipe = make_pipeline(oracle_nets, cuda_device, **params)
    if sinc_form == "window":
        window_form(pipe)
    cfg = pipe.config
    oracle = OraclePipeline(*oracle_nets, tau_active=cfg.tau_active, rho_update=cfg.rho_update,
                            delta_new=cfg.delta_new, max_speakers=cfg.max_speakers, as_reference=False)
    replay = OracleClustering(cfg.tau_active, cfg.rho_update, cfg.delta_new, "cosine", cfg.max_speakers)
    seg_err = emb_err = 0.0
    first_diff = None
    for b in range(N_CHUNKS // BATCH):
        x = torch.from_numpy(synth.windows(stream, BATCH, first=b * BATCH))
        seg, emb, maps = pipe.device_step(x.to(cuda_device))
        seg, emb, maps = seg.cpu().numpy(), emb.cpu().numpy(), maps.cpu().numpy()
        o_seg, o_emb, o_maps, margins = oracle(x)
        seg_err = max(seg_err, np.abs(seg - o_seg).max())
        emb_err = max(emb_err, np.abs(emb - o_emb).max())
        # (1) integer logic: oracle clustering replayed on the CUDA path's own scores / embeddings
        r_maps = np.stack([replay(s, e)[0] for s, e in zip(seg, emb)])
        assert np.array_equal(maps, r_maps), f"batch {b}: clustering kernel differs from the oracle on identical inputs"
        # (2) end to end
        if first_diff is None and not np.array_equal(maps, o_maps):
            i = int(np.where((maps != o_maps).any(axis=1))[0][0])
            first_diff = (b * BATCH + i, float(margins[i]))
    print(f"seg max abs err {seg_err:.2e}, emb max abs err {emb_err:.2e}, first end-to-end difference {first_diff}")
    assert seg_err < 1e-4 and emb_err < 1e-4
    if first_diff is not None:
        assert first_diff[1] < 1e-3, f"maps diverge at chunk {first_diff[0]} although the decision margin is {first_diff[1]}"
    assert np.array_equal(pipe.clustering.centers, replay.centers)


def test_speaker_diarization_drop_in(oracle_nets, stream, cuda_device):
    """SpeakerDiarization.__call__(Sequence[SlidingWindowFeature]) -> Sequence[(Annotation, SlidingWindowFeature)],
    the contract StreamingInference relies on (reference inference.py:137-141)."""
    pipe = make_pipeline(oracle_nets, cuda_device)
    host = make_pipeline(oracle_nets, cuda_device)          # same pipeline, fed through the per-block API
    sr, step, n = 16000, 0.5, 12
    chunks = [SlidingWindowFeature(stream[8000 * i:8000 * i + 80000, None],
                                   SlidingWindow(start=step * i, duration=1 / sr, step=1 / sr)) for i in range(n)]
    out = pipe(chunks[:5]) + pipe(chunks[5:])
    assert len(out) == n
    x = torch.from_numpy(synth.windows(stream, n))
    seg = host.segmentation(x[:, :, None])
    emb = host.embedding(x[:, :, None], seg)
    res = 5 / seg.shape[1]
    rttm_ref = []
    pred_buffer = []
    for i in range(n):
        swf = SlidingWindowFeature(seg[i].numpy(), SlidingWindow(start=step * i, duration=res, step=res))
        pred_buffer = [host.clustering(swf, emb[i])]
        rttm_ref.append(host.binarize(host.pred_aggregation(pred_buffer)).to_rttm())
    for i, (annotation, audio) in enumerate(out):
        assert annotation.to_rttm() == rttm_ref[i], f"chunk {i}"
        assert audio.data.shape[1] == 1 and 7999 <= audio.data.shape[0] <= 80000
    assert abs(out[0][1].extent.start) < 1e-9 and abs(out[3][1].extent.start - (3 * step + 4.5)) < 1e-3
    with pytest.raises(AssertionError):
        pipe([SlidingWindowFeature(stream[:1000, None], SlidingWindow(start=0, duration=1 / sr, step=1 / sr))])
    pipe.reset()
    assert pipe.clustering.centers is None


def test_call_uploads_a_stream_once_and_falls_back_for_anything_else(oracle_nets, cuda_device):
    """__call__ verifies on the host that the windows are consecutive hops of one stream and then uploads every sample once
    (dg_pipeline_call_host); a batch that breaks the pattern -- here: a jump inside the second sub-batch, and a batch of
    unrelated windows -- takes the full gather.  Both must give exactly what the fused step gives on the stacked windows."""
    from diart_b200 import _lib

    sr, step, n = 16000, 0.5, 72
    audio = synth.synth_audio(80000 + 8000 * (n + 40), seed=5)
    starts = [8000 * i for i in range(n)]
    jump = list(starts)
    for i in range(50, n):
        jump[i] += 8000 * 17 + 4000          # window 50 does not continue window 49
    shuffled = [starts[(7 * i) % n] for i in range(n)]
    for name, offs, expect_stream in (("stream", starts, True), ("jump", jump, False), ("shuffled", shuffled, False)):
        pipe = make_pipeline(oracle_nets, cuda_device)
        ref = make_pipeline(oracle_nets, cuda_device)
        chunks = [SlidingWindowFeature(np.ascontiguousarray(audio[o:o + 80000, None]),
                                       SlidingWindow(start=step * i, duration=1 / sr, step=1 / sr)) for i, o in enumerate(offs)]
        out = pipe(chunks)
        uploaded = int(_lib.lib().dg_pipeline_last_call_h2d_bytes(pipe._fused))
        if expect_stream:
            assert uploaded == (80000 + 8000 * (n - 1)) * 4, f"{name}: {uploaded} bytes uploaded"
        else:
            assert uploaded > n * 80000 * 4 // 3, f"{name}: {uploaded} bytes uploaded"
        x = torch.from_numpy(np.stack([audio[o:o + 80000] for o in offs])).to(cuda_device)
        seg, _, maps = ref.device_step(x)
        seg, maps = seg.cpu().numpy(), maps.cpu().numpy()
        res = 5 / seg.shape[1]
        for i in range(n):          # latency = step: every output is the binarised, permuted score of its own chunk
            permuted = np.zeros((seg.shape[1], ref.config.max_speakers))
            for k, g in enumerate(maps[i]):
                if g >= 0:
                    permuted[:, g] = seg[i][:, k]
            swf = SlidingWindowFeature(permuted, SlidingWindow(start=step * i, duration=res, step=res))
            want = ref.binarize(ref.pred_aggregation([swf])).to_rttm()
            if out[i][0].to_rttm() != want:
                # the reference step ran the whole batch through ONE form of the sinc layer, the call may have run its first
                # sub-batch through the stream form (scores differ by ~1e-5): only a score that close to the threshold may flip
                clearance = np.abs(permuted[permuted != 0] - ref.config.tau_active).min()
                assert not expect_stream and clearance < 2e-4, f"{name}: chunk {i} differs, threshold clearance {clearance:.1e}"


def test_call_refuses_a_bad_plan_before_touching_any_state(oracle_nets, stream, cuda_device):
    """dg_pipeline_call_host checks the plan rows at entry: a row whose buffers reach before the stream's first chunk is
    refused before any launch, and the calls after it give what a pipeline that never saw it gives"""
    import ctypes

    from diart_b200.blocks.post import post_plan

    pipe = make_pipeline(oracle_nets, cuda_device, latency=1.5)
    ref = make_pipeline(oracle_nets, cuda_device, latency=1.5)
    sr, step, n = 16000, 0.5, 12
    chunks = [SlidingWindowFeature(np.ascontiguousarray(stream[8000 * i:8000 * i + 80000, None]),
                                   SlidingWindow(start=step * i, duration=1 / sr, step=1 / sr)) for i in range(n)]
    h, F, K, _ = pipe._ensure_fused(80000)
    post = pipe._ensure_post(F, K)
    plan = np.ascontiguousarray(post_plan(np.arange(5) * step, 5 / F, np.zeros(0), np.zeros(0), post.nw, F, step, 1.5)[0])
    plan[1, 0] = 3
    header, turns = post.buffers(5)
    rows = (ctypes.c_void_p * 5)(*[c.data.ctypes.data for c in chunks[:5]])
    lib = _lib.lib()
    before = lib.dg_launch_count()
    rc = lib.dg_pipeline_call_host(h, post.handle, rows, 5, 80000, plan.ctypes.data, header.ctypes.data, turns.ctypes.data,
                                   len(turns), ctypes.byref(ctypes.c_int()), None, None)
    assert rc == -1 and lib.dg_launch_count() == before
    assert b"dg_pipeline_call_host: plan row 1 " in lib.dg_last_error()
    got = pipe(chunks[:5]) + pipe(chunks[5:])
    want = ref(chunks[:5]) + ref(chunks[5:])
    assert [a.to_rttm() for a, _ in got] == [a.to_rttm() for a, _ in want]
    assert sum(len(a.to_rttm()) for a, _ in got) > 0


def test_two_pipelines_on_the_same_model_handles(oracle_nets, stream, cuda_device):
    """two SpeakerDiarization instances built on the SAME SegmentationModel / EmbeddingModel objects (two audio streams, one set
    of weights) share the handles' activation buffers: submits of both in flight at once must hand the buffers over in stream order
    and give what each pipeline gives on its own"""
    seg_o, emb_o = oracle_nets
    seg_m = models.SegmentationModel(models.B200SegmentationLoader(seg_o.state_dict()))
    emb_m = models.EmbeddingModel(models.B200EmbeddingLoader(emb_o.state_dict()))
    mk = lambda: blocks.SpeakerDiarization(blocks.SpeakerDiarizationConfig(segmentation=seg_m, embedding=emb_m, device=cuda_device))
    a, b, ref = mk(), mk(), mk()
    xs = [torch.from_numpy(synth.windows(stream, BATCH, first=i * BATCH)).to(cuda_device) for i in range(3)]
    want = [[t.cpu().numpy() for t in ref.device_step(x)] for x in xs]          # ref sees batches 0, 1, 2 in order
    ref.reset()
    got_a, got_b = [], []
    for i in range(3):                      # a and b both see batches 0, 1, 2; their steps are interleaved and overlap
        a.submit(xs[i])
        b.submit(xs[i])
        if i > 0:
            got_a.append(a.collect())
            got_b.append(b.collect())
    got_a.append(a.collect())
    got_b.append(b.collect())
    torch.cuda.synchronize()
    for i in range(3):
        for name, w, ga, gb in zip(("seg", "emb", "map"), want[i], got_a[i], got_b[i]):
            assert np.array_equal(w, ga.cpu().numpy()), f"pipeline a, batch {i}: {name}"
            assert np.array_equal(w, gb.cpu().numpy()), f"pipeline b, batch {i}: {name}"


def test_foreign_models_behind_loader_api(oracle_nets, stream, cuda_device):
    """any Callable behind SegmentationModel / EmbeddingModel still works (block-by-block path);
    here: the oracle torch modules moved to the GPU"""
    import copy

    # torch's own GPU kernels default to TF32 convolutions (1e-3 error): compare against true float32
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    seg_o, emb_o = (copy.deepcopy(m) for m in oracle_nets)
    config = blocks.SpeakerDiarizationConfig(segmentation=models.SegmentationModel(lambda: seg_o),
                                             embedding=models.EmbeddingModel(lambda: emb_o), device=cuda_device)
    pipe = blocks.SpeakerDiarization(config)
    native = make_pipeline(oracle_nets, cuda_device)
    x = torch.from_numpy(synth.windows(stream, 4)).to(cuda_device)
    s1, e1, m1 = pipe.device_step(x)
    s2, e2, m2 = native.device_step(x)
    # torch's cuDNN / cuBLAS float32 kernels re-associate differently from both the CPU oracle and this path
    assert (s1 - s2).abs().max().item() < 1e-3 and (e1 - e2).abs().max().item() < 2e-3
    assert m1.shape == m2.shape and m1.dtype == torch.int32


def test_pipelined_submit_collect_equals_sequential_steps(oracle_nets, stream, cuda_device):
    """dg_pipeline_submit / collect (clustering of step i overlapping the networks of step i+1) must give exactly
    what one-step-at-a-time dg_pipeline_step gives: chunk order per stream is preserved"""
    a = make_pipeline(oracle_nets, cuda_device)
    b = make_pipeline(oracle_nets, cuda_device)
    nb = N_CHUNKS // 6     # six consecutive batches out of the 48-chunk stream
    batches = [torch.from_numpy(synth.windows(stream, nb, first=i * nb)).to(cuda_device) for i in range(6)]
    ref = [a.device_step(x) for x in batches]
    got = []
    b.submit(batches[0])
    b.submit(batches[1])
    got.append(b.collect())          # two outstanding (what bench.py's device loop does)
    b.submit(batches[2])
    b.submit(batches[3])             # three outstanding: slots 1, 2, 0 and lanes 1, 0, 1
    got.append(b.collect())
    b.submit(batches[4])
    got.append(b.collect())
    b.submit(batches[5])
    got.extend(b.collect() for _ in range(3))
    torch.cuda.synchronize()
    for (s1, e1, m1), (s2, e2, m2) in zip(ref, got):
        assert torch.equal(s1, s2) and torch.equal(e1, e2) and torch.equal(m1, m2)
    assert np.array_equal(a.clustering.centers, b.clustering.centers)
    with pytest.raises(ValueError):
        b.collect() if False else _lib_collect_empty(b)


def _lib_collect_empty(pipe):
    from diart_b200 import _lib

    _lib.check(_lib.lib().dg_pipeline_collect(pipe._fused, None, None, None, None))


def test_voice_activity_detection_pipeline(oracle_nets, stream, cuda_device):
    """VAD = max over local speakers of the same segmentation (reference blocks/vad.py:145-148)"""
    seg_o, _ = oracle_nets
    config = blocks.VoiceActivityDetectionConfig(
        segmentation=models.SegmentationModel(models.B200SegmentationLoader(seg_o.state_dict())), device=cuda_device)
    vad = blocks.VoiceActivityDetection(config)
    sr, n = 16000, 4
    chunks = [SlidingWindowFeature(stream[8000 * i:8000 * i + 80000, None],
                                   SlidingWindow(start=0.5 * i, duration=1 / sr, step=1 / sr)) for i in range(n)]
    out = vad(chunks)
    assert len(out) == n
    x = torch.from_numpy(synth.windows(stream, n))
    with torch.no_grad():
        ref = seg_o(x[:, None, :]).max(dim=-1, keepdim=True)[0].numpy()
    res = 5 / ref.shape[1]
    for i, (annotation, audio) in enumerate(out):
        swf = SlidingWindowFeature(ref[i], SlidingWindow(start=0.5 * i, duration=res, step=res))
        expect = Binarize(0.6)(blocks.DelayedAggregation(0.5, 0.5, "hamming", "loose")([swf]))
        got = sorted((round(s.start, 3), round(s.end, 3)) for s, _ in annotation.itertracks())
        want = sorted((round(s.start, 3), round(s.end, 3)) for s, _ in expect.itertracks())
        assert got == want and all(lab == "speech" for _, _, lab in annotation.itertracks(yield_label=True))
    # latency > step: the device aggregation over the 4 most recent chunks against the host mirrors of the reference's loop
    # (vad.py:150-190) fed with the SAME device scores
    cfg2 = blocks.VoiceActivityDetectionConfig(segmentation=config.segmentation, latency=2.0, device=cuda_device)
    vad2 = blocks.VoiceActivityDetection(cfg2)
    chunks2 = [SlidingWindowFeature(stream[8000 * i:8000 * i + 80000, None],
                                    SlidingWindow(start=0.5 * i, duration=1 / sr, step=1 / sr)) for i in range(9)]
    out2 = vad2(chunks2[:5]) + vad2(chunks2[5:])
    scores = vad2.segmentation.forward_device(torch.from_numpy(synth.windows(stream, 9)))
    host_scores = scores.amax(dim=-1, keepdim=True).cpu().numpy()
    agg, binarize, buf = blocks.DelayedAggregation(0.5, 2.0, "hamming", "loose"), Binarize(0.6), []
    for i in range(9):
        buf.append(SlidingWindowFeature(host_scores[i], SlidingWindow(start=0.5 * i, duration=res, step=res)))
        expect = binarize(agg(buf))
        got = sorted((s.start, s.end) for s, _ in out2[i][0].itertracks())
        want = sorted((s.start, s.end) for s, _ in expect.itertracks())
        assert got == want, f"latency 2.0, chunk {i}"
        if len(buf) == agg.num_overlapping_windows:
            buf = buf[1:]


def test_host_submit_collect_matches_step_host(oracle_nets, stream, cuda_device):
    """C ABI with HOST buffers: dg_pipeline_submit_host / collect_host (three steps outstanding) == dg_pipeline_step_host"""
    from diart_b200 import _lib

    lib = _lib.lib()
    a, b = make_pipeline(oracle_nets, cuda_device), make_pipeline(oracle_nets, cuda_device)
    ha, F, K, D = a._ensure_fused(80000)
    hb, _, _, _ = b._ensure_fused(80000)
    nb = N_CHUNKS // 6
    batches = [np.ascontiguousarray(synth.windows(stream, nb, first=i * nb)) for i in range(5)]

    def bufs():
        return (np.empty((nb, F, K), np.float32), np.empty((nb, K, D), np.float32), np.empty((nb, K), np.int32))

    ref = []
    for x in batches:
        s, e, m = bufs()
        _lib.check(lib.dg_pipeline_step_host(ha, x.ctypes.data, nb, 80000, s.ctypes.data, e.ctypes.data, m.ctypes.data, None))
        ref.append((s, e, m))
    got = []
    for x in batches[:3]:
        _lib.check(lib.dg_pipeline_submit_host(hb, x.ctypes.data, nb, 80000))
    assert lib.dg_pipeline_submit_host(hb, batches[3].ctypes.data, nb, 80000) == -1      # only three outstanding
    for nxt in (batches[3], batches[4], None, None, None):
        s, e, m = bufs()
        _lib.check(lib.dg_pipeline_collect_host(hb, s.ctypes.data, e.ctypes.data, m.ctypes.data))
        got.append((s, e, m))
        if nxt is not None:
            _lib.check(lib.dg_pipeline_submit_host(hb, nxt.ctypes.data, nb, 80000))
    assert lib.dg_pipeline_collect_host(hb, None, None, None) == -1                          # nothing outstanding
    for (s1, e1, m1), (s2, e2, m2) in zip(ref, got):
        assert np.array_equal(s1, s2) and np.array_equal(e1, e2) and np.array_equal(m1, m2)
