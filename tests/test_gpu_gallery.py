"""Gallery naming on the device: dg_gallery_query against the float64 oracle (tests/gallery_oracle.py) over gallery sizes
around the 64-entry tile and up to 100 000 entries, and MultiStreamDiarization with a gallery, whose labels after every tick
are the oracle's replayed on the streams' own centroids and whose turns are those of the same server without a gallery.

Models and audio are the seeded synthetic ones of diart_b200.synth."""
import numpy as np
import pytest
import torch

from diart_b200 import _lib, synth
from diart_b200.serve import MultiStreamDiarization
from diart_b200.speakers import KnownSpeakers, SpeakerGallery, speaker_labels
from gallery_oracle import cosine_distances, first_copies, name_step, nearest, resolve
from test_gpu_known_speakers import S, HOP, learned, make_config, states  # noqa: F401 (fixture)

pytestmark = pytest.mark.gpu

MARGIN = 1e-9


def query_case(G, D, Q, seed, threshold=0.25):
    """a gallery with duplicate rows, queries in contiguous groups of 1 .. 32 (random directions and queries planted near
    entries, two of a group sometimes near the same entry), and per group claimed entries (some of them planted targets)"""
    rng = np.random.default_rng(seed)
    E = rng.standard_normal((G, D)) * rng.uniform(0.5, 3.0, (G, 1))
    if G >= 8:
        src = rng.choice(G, size=max(2, G // 50), replace=False)
        dst = rng.choice(G, size=len(src), replace=False)
        E[dst] = E[src]
    X = rng.standard_normal((Q, D))
    target = rng.integers(0, G, Q)
    planted = rng.random(Q) < 0.6
    noise = rng.uniform(0.05, 0.6, Q)
    X[planted] = E[target[planted]] * rng.uniform(0.2, 5.0, (planted.sum(), 1)) + \
        noise[planted, None] * np.linalg.norm(E[target[planted]], axis=1, keepdims=True) / np.sqrt(D) * \
        rng.standard_normal((planted.sum(), D))
    sizes = []
    while sum(sizes) < Q:
        sizes.append(int(min(rng.integers(1, 33), Q - sum(sizes))))
    group = np.repeat(np.arange(len(sizes)), sizes).astype(np.int32)
    # some groups: a second query near the same entry as the first
    start = np.cumsum(sizes) - sizes
    for s0, n in zip(start, sizes):
        if n > 1 and rng.random() < 0.5 and planted[s0]:
            X[s0 + 1] = E[target[s0]] + 0.5 * noise[s0] * np.linalg.norm(E[target[s0]]) / np.sqrt(D) * rng.standard_normal(D)
            planted[s0 + 1] = True
            target[s0 + 1] = target[s0]
    claimed = np.full((len(sizes), 32), -1, dtype=np.int32)
    for r, (s0, n) in enumerate(zip(start, sizes)):
        k = int(rng.integers(0, 4))
        pick = list(rng.choice(G, size=min(k, G), replace=False))
        if rng.random() < 0.3 and planted[s0]:
            pick.append(int(target[s0]))
        pick = list(dict.fromkeys(pick))[:32]
        claimed[r, :len(pick)] = pick
    return E, X, group, claimed, threshold


def oracle_query(E, X, group, claimed, threshold):
    copies = first_copies(E)
    entry = np.full(len(X), -1, dtype=np.int64)
    best = np.empty(len(X))
    runner = np.empty(len(X))
    won = np.full(len(X), -1, dtype=np.int64)
    for r in np.unique(group):
        rows = np.flatnonzero(group == r)
        d = cosine_distances(X[rows], E, copies)
        e, b, run = nearest(d, [c for c in claimed[r] if c >= 0])
        entry[rows], best[rows], runner[rows] = e, b, run
        won[rows] = resolve(e, b, threshold)
    return entry, best, runner, won


def comparable(entry, best, runner, group, threshold):
    """queries whose outcome no rounding can change: best more than MARGIN from the threshold, from the runner-up, and from
    any other candidate of its group for the same entry"""
    with np.errstate(invalid="ignore"):
        ok = ~np.isfinite(best) | ((np.abs(best - threshold) > MARGIN) & ((runner - best) > MARGIN))
    for q in range(len(entry)):
        same = (group == group[q]) & (entry == entry[q]) & (np.arange(len(entry)) != q)
        if entry[q] >= 0 and np.any(np.abs(best[same] - best[q]) <= MARGIN):
            ok[q] = False
    return ok


@pytest.mark.parametrize("G,D,Q", [(1, 256, 1), (1, 512, 40), (127, 512, 700), (128, 256, 300), (129, 512, 2500),
                                   (10000, 512, 3000), (10000, 256, 1200), (100000, 512, 300), (100000, 256, 160)])
def test_query_equals_the_float64_oracle(cuda_device, G, D, Q):
    E, X, group, claimed, threshold = query_case(G, D, Q, seed=G * 7 + D + Q)
    gal = SpeakerGallery(KnownSpeakers([f"p{i}" for i in range(G)], E), threshold, cuda_device)
    x_d = torch.from_numpy(X).to(cuda_device)
    g_d = torch.from_numpy(group).to(cuda_device)
    c_d = torch.from_numpy(claimed).to(cuda_device)
    e_d = torch.empty(Q, dtype=torch.int32, device=cuda_device)
    d_d = torch.empty(Q, dtype=torch.float64, device=cuda_device)
    _lib.check(_lib.lib().dg_gallery_query(gal.handle, x_d.data_ptr(), Q, g_d.data_ptr(), c_d.data_ptr(), threshold,
                                           e_d.data_ptr(), d_d.data_ptr(), _lib.stream_ptr(cuda_device)))
    got_e, got_d = e_d.cpu().numpy(), d_d.cpu().numpy()
    entry, best, runner, won = oracle_query(E, X, group, claimed, threshold)
    fin = np.isfinite(best)
    assert np.array_equal(np.isfinite(got_d), fin)
    assert np.abs(got_d[fin] - best[fin]).max(initial=0.0) <= 1e-12
    ok = comparable(entry, best, runner, group, threshold)
    assert ok.all(), f"{(~ok).sum()} queries inside the margin: the generator must keep them away"
    assert np.array_equal(got_e, won)
    if G > 1:
        assert (won >= 0).sum() > 0 and (won < 0).sum() > 0
    # identical rows give identical distances, so the lowest copy the group has not claimed is chosen
    first = first_copies(E)
    for q in np.flatnonzero(won >= 0):
        lower = np.flatnonzero((first == first[won[q]]) & (np.arange(G) < won[q]))
        assert np.isin(lower, claimed[group[q]]).all(), (q, won[q], lower)
    # the claims were honoured
    for q in np.flatnonzero(won >= 0):
        assert won[q] not in claimed[group[q]]


def test_query_refusals(cuda_device):
    gal = SpeakerGallery(KnownSpeakers(["a", "b"], np.eye(2, 4)), 0.5, cuda_device)
    x = torch.ones((3, 4), dtype=torch.float64, device=cuda_device)
    e = torch.empty(3, dtype=torch.int32, device=cuda_device)
    d = torch.empty(3, dtype=torch.float64, device=cuda_device)
    lib = _lib.lib()
    for groups in ([0, 1, 0], [0, -1, 1]):
        g = torch.tensor(groups, dtype=torch.int32, device=cuda_device)
        assert lib.dg_gallery_query(gal.handle, x.data_ptr(), 3, g.data_ptr(), None, 0.5, e.data_ptr(), d.data_ptr(),
                                    _lib.stream_ptr(cuda_device)) == -1
    g = torch.zeros(33, dtype=torch.int32, device=cuda_device)
    x33 = torch.ones((33, 4), dtype=torch.float64, device=cuda_device)
    assert lib.dg_gallery_query(gal.handle, x33.data_ptr(), 33, g.data_ptr(), None, 0.5, e.data_ptr(), d.data_ptr(),
                                _lib.stream_ptr(cuda_device)) == -1
    assert b"more than 32" in lib.dg_last_error()
    g = torch.zeros(3, dtype=torch.int32, device=cuda_device)
    for t in (0.0, 2.5, float("nan")):
        assert lib.dg_gallery_query(gal.handle, x.data_ptr(), 3, g.data_ptr(), None, t, e.data_ptr(), d.data_ptr(),
                                    _lib.stream_ptr(cuda_device)) == -1


def test_identify_and_name(cuda_device):
    rng = np.random.default_rng(5)
    E = rng.standard_normal((500, 512))
    gal = SpeakerGallery(KnownSpeakers([f"p{i}" for i in range(500)], E), 0.1, cuda_device)
    X = np.stack([E[7] * 3 + 0.01 * rng.standard_normal(512), E[9], rng.standard_normal(512)])
    entry, dist = gal.identify(X)
    assert entry.tolist() == [7, 9, -1] and dist.dtype == np.float64 and abs(dist[1]) <= 1e-12
    assert gal.identify(X, claimed=[7])[0].tolist() == [-1, 9, -1]
    state = KnownSpeakers(["p9", "speaker1", "speaker2", "speaker3"], np.stack([E[9], E[9] * 2, X[0], X[2]]))
    named = gal.name(state)
    assert named.names == ("p9", "speaker1", "p7", "speaker3")
    assert np.array_equal(named.centroids, state.centroids)
    assert gal.name(named) == named


def drive(server, audio, plan, gallery, rng_seed, resume_at=None):
    """opens plan[k] = (open kwargs) at tick 0, pushes ragged blocks to every stream and ticks until the audio is consumed;
    at tick ``resume_at`` stream 0 is closed and reopened from speakers().  -> per tick: {key: (labels after the tick,
    centroids, RTTM lines of the tick's annotations)}"""
    rng = np.random.default_rng(rng_seed)
    sid = {k: server.open(**kw) for k, kw in enumerate(plan)}
    pos = {k: 0 for k in sid}
    ticks = []
    tick = 0
    while any(pos[k] < len(audio[k]) for k in sid) or any(server.available(s) for s in sid.values()):
        if tick == resume_at:
            state = server.speakers(sid[0])
            server.close(sid[0])
            sid[0] = server.open(speakers=state)
            assert server.speakers(sid[0]).names == state.names
            pos[0] = max(0, pos[0] - S)          # a fresh ring: give the new stream a window's worth again
        for k, s in sid.items():
            n = int(rng.integers(0, 3 * HOP))
            block = audio[k][pos[k]:pos[k] + n]
            if len(block):
                server.push(s, block)
            pos[k] += len(block)
        res = server.step()
        tick += 1
        rec = {}
        key_of = {s: k for k, s in sid.items()}
        for s, anns in res.items():
            state = server.speakers(s)
            rec[key_of[s]] = (list(state.names), state.centroids, [a.to_rttm() for a in anns])
        ticks.append(rec)
    return ticks


def turns_by_index(rttm_lines, labels):
    """RTTM turns with each label replaced by its global speaker index"""
    index = {label: g for g, label in enumerate(labels)}
    out = []
    for text in rttm_lines:
        rows = []
        for line in text.splitlines():
            f = line.split()
            rows.append((f[3], f[4], index[f[7]]))
        out.append(rows)
    return out


def test_streams_are_named_from_a_large_gallery(states, cuda_device):
    config = make_config(states, cuda_device, latency=1.0)
    seeds = [3101, 3102, 3103, 3104]
    audio = {k: synth.synth_audio(S + HOP * 26, seed=s) for k, s in enumerate(seeds)}
    people = {k: learned(config, s, [f"p{k}a", f"p{k}b"]) for k, s in enumerate(seeds)}
    D = people[0].dimension
    rng = np.random.default_rng(77)
    decoys = rng.standard_normal((12000, D))
    # stream 2 starts from a known speaker who is also in the gallery; stream 3 from one who is not
    seed2 = KnownSpeakers(["p2a"], people[2].centroids[:1])
    seed3 = KnownSpeakers(["zed"], people[3].centroids[:1])
    plan = [dict(), dict(latency=2.0), dict(speakers=seed2), dict(speakers=seed3)]
    # the enrolled people: the first two speakers of every stream's audio, hidden among the decoys
    entries, names = [], []
    for k in range(4):
        for j in range(2):
            entries.append(people[k].centroids[j])
            names.append(people[k].names[j])
    at = np.sort(rng.choice(len(decoys) + len(entries), size=len(entries), replace=False))
    table = np.empty((len(decoys) + len(entries), D))
    mask = np.zeros(len(table), dtype=bool)
    mask[at] = True
    table[mask] = np.stack(entries)
    table[~mask] = decoys
    all_names = np.empty(len(table), dtype=object)
    all_names[mask] = names
    all_names[~mask] = [f"decoy{i}" for i in range(len(decoys))]
    all_names = list(all_names)

    base_server = MultiStreamDiarization(config, max_streams=6, max_windows_per_stream=3, max_latency=2.0)
    base = drive(base_server, audio, plan, None, 5, resume_at=9)
    # the threshold: halfway inside the widest gap among the distances of every state of the run to the enrolled people,
    # below 0.8 -- no distance is near it, and some speakers are named and others are not
    d = np.concatenate([cosine_distances(c, np.stack(entries)).min(axis=1) for rec in base for _, c, _ in rec.values()])
    d = np.unique(d[d < 0.8])
    gap = int(np.argmax(np.diff(d)))
    threshold = float((d[gap] + d[gap + 1]) / 2)
    assert d[gap + 1] - d[gap] > 1e-3, d

    gallery = SpeakerGallery(KnownSpeakers(all_names, table), threshold, cuda_device)
    server = MultiStreamDiarization(config, max_streams=6, max_windows_per_stream=3, max_latency=2.0, gallery=gallery)
    got = drive(server, audio, plan, gallery, 5, resume_at=9)
    assert len(got) == len(base)
    copies = first_copies(table)
    oracle = {k: list(speaker_labels(kw.get("speakers"), config.max_speakers)) for k, kw in enumerate(plan)}
    compared = 0
    for t, (rec, brec) in enumerate(zip(got, base)):
        assert rec.keys() == brec.keys(), f"tick {t}"
        for k, (labels, centroids, rttm) in rec.items():
            b_labels, b_centroids, b_rttm = brec[k]
            assert np.array_equal(centroids.view(np.int64), b_centroids.view(np.int64)), f"tick {t} stream {k}"
            want, cmp = name_step(oracle[k][:len(labels)], centroids, all_names, table, threshold, copies)
            for g, best, runner, margin in cmp:
                assert margin > MARGIN and runner - best > MARGIN, (t, k, g)
            compared += len(cmp)
            oracle[k][:len(labels)] = want
            assert labels == want, f"tick {t} stream {k}"
            # names change labels, never segments
            assert turns_by_index(rttm, labels) == turns_by_index(b_rttm, b_labels + [f"speaker{g}" for g in
                                                                                     range(len(b_labels), 32)]), (t, k)
    final = {k: oracle[k] for k in oracle}
    active = {k: max(len(rec[k][0]) for rec in got if k in rec) for k in final}
    assert compared > 0 and any(label in names for k in final for label in final[k]), final
    assert any(final[k][g] == f"speaker{g}" for k in final for g in range(active[k])), "every speaker was named"
    assert final[2][0] == "p2a" and final[3][0] == "zed"
    assert "p2a" not in final[2][1:], "a claimed entry named a second speaker"
