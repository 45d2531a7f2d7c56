"""Synchronous and submitted steps of one fused pipeline handle.

dg_pipeline_step, dg_pipeline_step_host and dg_pipeline_call_stream enqueue a step on scratch lane 0 without a result slot;
the dg_pipeline_submit* steps rotate through three slots and two lanes.  Both kinds share lane 0, the clustering stream and
the clustering state.  These tests mix them on one handle and check:

- every step's results bit for bit against one-step-at-a-time execution on a fresh pipeline, and that a synchronous step
  leaves the slot buffers a dg_pipeline_collect handed out untouched;
- the permuted scores of the synchronous steps against SpeakerMap.apply of that step's scores and map;
- that a synchronous step is refused while a submitted step is outstanding, and leaves the handle usable."""
import ctypes as C

import numpy as np
import pytest
import torch

from diart_b200 import _lib, blocks, models, synth
from diart_b200.mapping import SpeakerMap
from diart_b200.operators import DeviceAudioStream

pytestmark = pytest.mark.gpu
NB, S = 8, 80000


@pytest.fixture(scope="module")
def stream():
    return synth.synth_audio(S + 8000 * (7 * NB - 1), seed=777, num_speakers=4)


def make_pipeline(oracle_nets, device):
    seg_o, emb_o = oracle_nets
    config = blocks.SpeakerDiarizationConfig(
        segmentation=models.SegmentationModel(models.B200SegmentationLoader(seg_o.state_dict())),
        embedding=models.EmbeddingModel(models.B200EmbeddingLoader(emb_o.state_dict())), device=device)
    return blocks.SpeakerDiarization(config)


class _DeviceView:
    """a device buffer owned by the library, seen by torch without a copy"""

    def __init__(self, ptr, shape, typestr):
        self.__cuda_array_interface__ = {"data": (ptr, False), "shape": shape, "typestr": typestr, "strides": None,
                                         "version": 2}


def collect_views(lib, h, B, F, K, D, device):
    """dg_pipeline_collect: the oldest submitted step's slot buffers (valid until the third next submit), ordered on the
    current stream"""
    p = [C.c_void_p() for _ in range(3)]
    _lib.check(lib.dg_pipeline_collect(h, C.byref(p[0]), C.byref(p[1]), C.byref(p[2]), _lib.stream_ptr(device)))
    return [torch.as_tensor(_DeviceView(q.value, shape, t), device=device)
            for q, shape, t in zip(p, ((B, F, K), (B, K, D), (B, K)), ("<f4", "<f4", "<i4"))]


def test_sync_steps_between_submitted_steps(oracle_nets, stream, cuda_device):
    """submit, submit, collect, collect, dg_pipeline_step, dg_pipeline_step_host, then three submit_host with their collects,
    all on one handle, == device_step over the same batches on a fresh pipeline"""
    lib = _lib.lib()
    ref, pipe = make_pipeline(oracle_nets, cuda_device), make_pipeline(oracle_nets, cuda_device)
    h, F, K, D = pipe._ensure_fused(S)
    M = pipe.config.max_speakers
    sp = _lib.stream_ptr(cuda_device)
    xs = [np.ascontiguousarray(synth.windows(stream, NB, first=i * NB)) for i in range(7)]
    dev = [torch.from_numpy(x).to(cuda_device) for x in xs]
    want = [[t.cpu().numpy() for t in ref.device_step(x)] for x in dev]

    def host_bufs():
        return np.empty((NB, F, K), np.float32), np.empty((NB, K, D), np.float32), np.empty((NB, K), np.int32)

    got, perms = [], []
    for x in dev[:2]:                                  # slots 0, 1; lanes 0, 1
        _lib.check(lib.dg_pipeline_submit(h, x.data_ptr(), NB, S, sp))
    views = [collect_views(lib, h, NB, F, K, D, cuda_device) for _ in range(2)]
    got += [[v.cpu().numpy() for v in vs] for vs in views]
    kept = [v.clone() for v in views[1]]

    seg, emb = torch.empty((NB, F, K), device=cuda_device), torch.empty((NB, K, D), device=cuda_device)
    maps, perm = torch.empty((NB, K), dtype=torch.int32, device=cuda_device), torch.empty((NB, F, M), device=cuda_device)
    _lib.check(lib.dg_pipeline_step(h, dev[2].data_ptr(), NB, S, seg.data_ptr(), emb.data_ptr(), maps.data_ptr(),
                                    perm.data_ptr(), sp))
    got.append([seg.cpu().numpy(), emb.cpu().numpy(), maps.cpu().numpy()])
    perms.append(perm.cpu().numpy())
    for name, v, k in zip(("seg", "emb", "map"), views[1], kept):
        assert torch.equal(v, k), f"dg_pipeline_step changed the collected step's {name}"

    s, e, m = host_bufs()
    p = np.empty((NB, F, M), np.float32)
    _lib.check(lib.dg_pipeline_step_host(h, xs[3].ctypes.data, NB, S, s.ctypes.data, e.ctypes.data, m.ctypes.data,
                                         p.ctypes.data))
    got.append([s, e, m])
    perms.append(p)
    for name, v, k in zip(("seg", "emb", "map"), views[1], kept):
        assert torch.equal(v, k), f"dg_pipeline_step_host changed the collected step's {name}"

    for x in xs[4:]:                                   # slots 2, 0, 1; lanes 0, 1, 0: the rotation goes on from the submits
        _lib.check(lib.dg_pipeline_submit_host(h, x.ctypes.data, NB, S))
    for _ in range(3):
        s, e, m = host_bufs()
        _lib.check(lib.dg_pipeline_collect_host(h, s.ctypes.data, e.ctypes.data, m.ctypes.data))
        got.append([s, e, m])
    torch.cuda.synchronize()

    for i, (w, g) in enumerate(zip(want, got)):
        for name, a, b in zip(("seg", "emb", "map"), w, g):
            assert np.array_equal(a, b), f"batch {i}: {name}"
    assert np.array_equal(ref.clustering.centers, pipe.clustering.centers)
    # permuted scores of the synchronous steps (permuted_dev, permuted_host): SpeakerMap.apply of the step's scores and map
    for (seg_b, _, map_b), perm_b in zip(got[2:4], perms):
        for s_w, m_w, p_w in zip(seg_b, map_b, perm_b):
            assert np.array_equal(p_w.astype(np.float64), SpeakerMap(m_w, M).apply(s_w))


def test_sync_steps_refused_while_a_submitted_step_is_outstanding(oracle_nets, stream, cuda_device):
    """dg_pipeline_step and dg_pipeline_call_stream return -1 while a submitted step is outstanding and enqueue nothing:
    after the collect, the handle gives what a pipeline that never saw the refused calls gives"""
    lib = _lib.lib()
    ref, pipe = make_pipeline(oracle_nets, cuda_device), make_pipeline(oracle_nets, cuda_device)
    h, F, K, D = pipe._ensure_fused(S)
    sp = _lib.stream_ptr(cuda_device)
    x = torch.from_numpy(synth.windows(stream, NB)).to(cuda_device)
    streams = []
    for _ in range(2):
        st = DeviceAudioStream(5, 0.5, 16000, max_windows=NB, device=cuda_device)
        st.push(stream[NB * 8000:NB * 8000 + S + 8000 * (NB - 1)])
        streams.append(st)
    want = [t.cpu().numpy() for t in ref.device_step(x)]

    pipe.submit(x)
    seg, emb = torch.empty((NB, F, K), device=cuda_device), torch.empty((NB, K, D), device=cuda_device)
    maps = torch.empty((NB, K), dtype=torch.int32, device=cuda_device)
    assert lib.dg_pipeline_step(h, x.data_ptr(), NB, S, seg.data_ptr(), emb.data_ptr(), maps.data_ptr(), None, sp) == -1
    assert "outstanding" in lib.dg_last_error().decode()
    post = pipe._ensure_post(F, K)
    plan = np.zeros((NB, 4 + post.nw), np.int32)
    header, turns = post.buffers(NB)
    n_turns = C.c_int()
    assert lib.dg_pipeline_call_stream(h, post.handle, streams[0].handle, NB, plan.ctypes.data, header.ctypes.data,
                                       turns.ctypes.data, len(turns), C.byref(n_turns), None, None) == -1
    assert "outstanding" in lib.dg_last_error().decode()
    assert streams[0].available == NB

    got = [t.cpu().numpy() for t in pipe.collect()]
    for name, a, b in zip(("seg", "emb", "map"), want, got):
        assert np.array_equal(a, b), name
    out, out_ref = pipe.call_stream(streams[0], NB), ref.call_stream(streams[1], NB)
    assert [a.to_rttm() for a, _ in out] == [a.to_rttm() for a, _ in out_ref]
    assert np.array_equal(ref.clustering.centers, pipe.clustering.centers)
