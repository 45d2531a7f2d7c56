"""Variant B of the embedding row (SURVEY.md 8(a) A8'): pyannote/wespeaker-voxceleb-resnet34-LM on the GPU -- kaldi fbank as a
wgmma GEMM over an overlapping-row view of the waveform, ResNet34 as shifted-window Conv2d GEMMs on zero-padded channels-last
maps (csrc/resnet.cu, TC_CONV2D epilogue of csrc/gemm_tc.cu) -- against the oracle restatement oracle.nets.WeSpeakerResNet34
(pinned by parameter count and map sizes in tests/test_oracle_golden.py).  Bar: unit-norm embeddings 1e-4 (the bar of
variant A); the stages against float64 are in tests/test_zz_wespeaker_stages.py."""
import numpy as np
import pytest
import torch

from diart_b200 import _lib, blocks, models, synth
from oracle import nets
from oracle.clustering import OracleClustering

N = 3


@pytest.fixture(scope="module")
def wespeaker():
    torch.set_num_threads(16)
    return nets.make_wespeaker()


@pytest.fixture(scope="module")
def audio():
    return torch.from_numpy(synth.windows(synth.synth_audio(80000 + 8000 * (N - 1), seed=99), N))


def test_variant_is_recognised_without_gpu():
    lib = _lib.lib()
    assert hasattr(lib, "dg_emb_debug_trunk")
    assert lib.dg_emb_debug_trunk(None, None, 1, 80000, 0, None, 0, None) == -1


@pytest.mark.gpu
def test_wespeaker_embeddings_match_oracle(wespeaker, audio, cuda_device):
    emb = models.B200EmbeddingLoader(wespeaker.state_dict())().to(cuda_device)
    g = torch.Generator().manual_seed(3)
    w = torch.rand((N, 293, 3), generator=g) ** 3
    with torch.no_grad():
        ref = wespeaker.forward_dedup(audio[:, None, :], w)
        ref_n = ref / ref.norm(dim=-1, keepdim=True)
    nrm = emb.forward_fused(audio.to(cuda_device), w.to(cuda_device), normalize=True).cpu()
    err = (nrm - ref_n).abs().max().item()
    print(f"WeSpeaker unit-norm embeddings: max abs err {err:.2e}")
    assert err < 1e-4
    # the reference's call convention: rows repeated once per local speaker, weights (N*K, F)
    rep = audio[:, None, :].repeat(1, 3, 1).reshape(N * 3, 1, -1)
    rows = emb(rep.to(cuda_device), w.permute(0, 2, 1).reshape(N * 3, 293).to(cuda_device)).reshape(N, 3, -1).cpu()
    raw = emb.forward_fused(audio.to(cuda_device), w.to(cuda_device)).cpu()
    assert torch.equal(rows, raw)
    plain = emb(audio[:, None, :].to(cuda_device), None).cpu()
    with torch.no_grad():
        ref_plain = wespeaker(audio[:, None, :], None)
    assert ((plain - ref_plain).norm(dim=-1) / ref_plain.norm(dim=-1)).max().item() < 3e-4


@pytest.mark.gpu
def test_pipeline_with_wespeaker_embedding(wespeaker, oracle_nets, cuda_device):
    """the fused step with variant B behind the same EmbeddingModel loader: scores / embeddings against the oracle networks,
    speaker maps identical to the oracle clustering replayed on them"""
    seg_o, _ = oracle_nets
    config = blocks.SpeakerDiarizationConfig(
        segmentation=models.SegmentationModel(models.B200SegmentationLoader(seg_o.state_dict())),
        embedding=models.EmbeddingModel(models.B200EmbeddingLoader(wespeaker.state_dict())), device=cuda_device)
    pipe = blocks.SpeakerDiarization(config)
    n = 12
    stream = synth.synth_audio(80000 + 8000 * (n - 1), seed=4242, num_speakers=4)
    x = torch.from_numpy(synth.windows(stream, n))
    seg, emb, maps = (t.cpu().numpy() for t in pipe.device_step(x.to(cuda_device)))
    assert emb.shape == (n, 3, 256)
    from oracle.pipeline import osp_block

    with torch.no_grad():
        o_seg = seg_o(x[:, None, :])
        o_emb = wespeaker.forward_dedup(x[:, None, :], osp_block(o_seg))
        o_emb = (o_emb / o_emb.norm(dim=-1, keepdim=True)).numpy()
    assert np.abs(seg - o_seg.numpy()).max() < 1e-4
    print(f"pipeline (variant B) emb max abs err {np.abs(emb - o_emb).max():.2e}")
    assert np.abs(emb - o_emb).max() < 1e-4
    replay = OracleClustering(0.6, 0.3, 1.0, "cosine", 20)
    want = np.stack([replay(s, e)[0] for s, e in zip(seg, emb)])
    assert np.array_equal(maps, want)
    assert np.array_equal(pipe.clustering.centers, replay.centers)
