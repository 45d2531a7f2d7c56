"""Per-stream galleries on the device: MultiStreamDiarization streams named from their own galleries and thresholds in one
grouped search per tick.  Labels after every tick are the float64 oracle's (tests/gallery_oracle.py) on the stream's own
gallery, and SpeakerGallery.name on the stream's previous labels and new centroids (the same kernel) reproduces them bit for
bit; turns are those of the same server without galleries.

Models and audio are the seeded synthetic ones of diart_b200.synth."""
import numpy as np
import pytest
import torch

from diart_b200 import _lib, blocks, synth
from diart_b200.serve import MultiStreamDiarization, MultiStreamVoiceActivityDetection
from diart_b200.speakers import KnownSpeakers, SpeakerGallery, speaker_labels
from gallery_oracle import cosine_distances, first_copies, name_step
from test_gpu_gallery import MARGIN, turns_by_index
from test_gpu_known_speakers import S, HOP, learned, make_config, states  # noqa: F401 (fixture)

pytestmark = pytest.mark.gpu


def drive(server, audio, plan, rng_seed, resume=None, launches=None):
    """opens plan[k] (open kwargs) at tick 0, pushes ragged blocks to every stream and ticks until the audio is consumed;
    resume = (tick, key): that stream is closed then and reopened from speakers() with its open kwargs' gallery.
    launches: a list that receives each tick's kernel launch count.  -> per tick {key: (labels, centroids, RTTM lines)}"""
    lib = _lib.lib()
    rng = np.random.default_rng(rng_seed)
    sid = {k: server.open(**kw) for k, kw in enumerate(plan)}
    pos = {k: 0 for k in sid}
    ticks = []
    while any(pos[k] < len(audio[k]) for k in sid) or any(server.available(s) for s in sid.values()):
        if resume is not None and len(ticks) == resume[0]:
            k = resume[1]
            state = server.speakers(sid[k])
            server.close(sid[k])
            sid[k] = server.open(speakers=state, **{a: v for a, v in plan[k].items() if a == "gallery"})
            assert server.speakers(sid[k]).names == state.names
            pos[k] = max(0, pos[k] - S)
        for k, s in sid.items():
            block = audio[k][pos[k]:pos[k] + int(rng.integers(0, 3 * HOP))]
            if len(block):
                server.push(s, block)
            pos[k] += len(block)
        before = lib.dg_launch_count()
        res = server.step()
        if launches is not None:
            launches.append(lib.dg_launch_count() - before)
        key_of = {s: k for k, s in sid.items()}
        rec = {}
        for s, anns in res.items():
            state = server.speakers(s)
            rec[key_of[s]] = (list(state.names), state.centroids, [a.to_rttm() for a in anns])
        ticks.append(rec)
    return ticks


def hidden(people, decoys, rng):
    """entries: people (names, rows) at random places among the decoy rows -> (names, table)"""
    names, rows = people
    n = len(decoys) + len(rows)
    at = np.sort(rng.choice(n, size=len(rows), replace=False))
    mask = np.zeros(n, dtype=bool)
    mask[at] = True
    table = np.empty((n, decoys.shape[1]))
    table[mask] = rows
    table[~mask] = decoys
    all_names = np.empty(n, dtype=object)
    all_names[mask] = list(names)
    all_names[~mask] = [f"decoy{i}" for i in range(len(decoys))]
    return list(all_names), table


def gap_threshold(base, key, people_rows):
    """halfway inside the widest gap below 0.8 among the distances of stream `key`'s states in the run to its people (half
    the nearest distance when fewer than two lie below 0.8), so that no distance is near it"""
    d = np.concatenate([cosine_distances(rec[key][1], people_rows).min(axis=1) for rec in base if key in rec])
    low = np.unique(d[d < 0.8])
    if len(low) < 2:
        return float(min(0.8, d.min()) / 2)
    gap = int(np.argmax(np.diff(low)))
    assert low[gap + 1] - low[gap] > 1e-3, low
    return float((low[gap] + low[gap + 1]) / 2)


def check_run(got, base, plan, galleries, config, seeded_names):
    """every tick: labels are the oracle's on the stream's own gallery (None: never named), the gallery's own kernel replays
    them bit for bit, no label comes from elsewhere, and the turns are the gallery-free server's"""
    oracle = {k: list(speaker_labels(kw.get("speakers"), config.max_speakers)) for k, kw in enumerate(plan)}
    copies = {k: first_copies(g.known.centroids) for k, g in galleries.items() if g is not None}
    compared = 0
    assert len(got) == len(base)
    for t, (rec, brec) in enumerate(zip(got, base)):
        assert rec.keys() == brec.keys(), f"tick {t}"
        for k, (labels, centroids, rttm) in rec.items():
            b_labels, b_centroids, b_rttm = brec[k]
            assert np.array_equal(centroids.view(np.int64), b_centroids.view(np.int64)), f"tick {t} stream {k}"
            g = galleries[k]
            prev = oracle[k][:len(labels)]
            if g is None:
                want = prev
            else:
                want, cmp = name_step(prev, centroids, g.names, g.known.centroids, g.threshold, copies[k])
                for q, best, runner, margin in cmp:
                    assert margin > MARGIN and runner - best > MARGIN, (t, k, q)
                compared += len(cmp)
                # the same kernel on the stream's previous labels and new centroids: bit for bit
                assert list(g.name(KnownSpeakers(prev, centroids)).names) == labels, f"tick {t} stream {k}"
            oracle[k][:len(labels)] = want
            assert labels == want, f"tick {t} stream {k}"
            own = set(g.names) if g is not None else set()
            for q, label in enumerate(labels):
                assert label == f"speaker{q}" or label in own or label in seeded_names.get(k, ()), (t, k, label)
            assert turns_by_index(rttm, labels) == turns_by_index(
                b_rttm, b_labels + [f"speaker{q}" for q in range(len(b_labels), 32)]), (t, k)
    return oracle, compared


def test_streams_named_from_their_own_galleries(states, cuda_device):
    config = make_config(states, cuda_device, latency=1.0)
    seeds = [4101, 4102, 4103, 4104, 4105, 4106]
    audio = {k: synth.synth_audio(S + HOP * 24, seed=s) for k, s in enumerate(seeds)}
    people = {k: learned(config, s, [f"p{k}a", f"p{k}b"]) for k, s in enumerate(seeds)}
    D = people[0].dimension
    rng = np.random.default_rng(91)
    seed2 = KnownSpeakers(["p2a"], people[2].centroids[:1])
    # the plan without galleries: stream 0 is resumed at tick 8, stream 2 is seeded, stream 1 has a longer latency
    bare = [dict(), dict(latency=2.0), dict(speakers=seed2), dict(), dict(), dict()]
    base_server = MultiStreamDiarization(config, max_streams=8, max_windows_per_stream=3, max_latency=2.0)
    base = drive(base_server, audio, bare, 5, resume=(8, 0))
    thr = {k: gap_threshold(base, k, people[k].centroids) for k in range(6)}
    assert len(set(round(v, 6) for v in thr.values())) > 1, thr
    # two tenants who both have an "alice" (different people); each also holds the other's people under foreign names
    a, b = people[0].centroids, people[1].centroids
    tenant_a = SpeakerGallery(KnownSpeakers(["alice", "bob", "b_alice", "b_carol"] + [f"a{i}" for i in range(60)],
                                            np.concatenate([a, b, rng.standard_normal((60, D))])), thr[0], cuda_device)
    tenant_b = SpeakerGallery(KnownSpeakers(["alice", "carol", "a_alice", "a_bob"] + [f"b{i}" for i in range(100)],
                                            np.concatenate([b, a, rng.standard_normal((100, D))])), thr[1], cuda_device)
    names, table = hidden((people[2].names, people[2].centroids), rng.standard_normal((12006, D)), rng)
    large = SpeakerGallery(KnownSpeakers(names, table), thr[2], cuda_device)
    names, table = hidden((people[3].names, people[3].centroids), rng.standard_normal((14, D)), rng)
    roster = SpeakerGallery(KnownSpeakers(names, table), thr[3], cuda_device)
    names, table = hidden((people[4].names, people[4].centroids), rng.standard_normal((500, D)), rng)
    default = SpeakerGallery(KnownSpeakers(names, table), thr[4], cuda_device)
    assert len(large) == 12008 and len(roster) == 16
    own = [tenant_a, tenant_b, large, roster, None, None]   # stream 4: the server's default; stream 5: none
    plan = [dict(kw, **({"gallery": g} if g is not None else {})) for kw, g in zip(bare, own)]
    seeded = {2: {"p2a"}}

    server = MultiStreamDiarization(config, max_streams=8, max_windows_per_stream=3, max_latency=2.0, gallery=default)
    got = drive(server, audio, plan, 5, resume=(8, 0))
    galleries = dict(enumerate(own[:4] + [default, default]))
    final, compared = check_run(got, base, plan, galleries, config, seeded)
    assert compared > 0
    # names were given, and each tenant's streams only ever carry that tenant's names (checked at every tick above)
    assert any(label in people[k].names for k in (2, 3, 4) for label in final[k]), final
    assert any(label in tenant_a.names for label in final[0]) and any(label in tenant_b.names for label in final[1]), final
    assert final[2][0] == "p2a" and "p2a" not in final[2][1:]

    # the same streams on a server without a default gallery: stream 4 stays unnamed, the others are named as before
    plain = MultiStreamDiarization(config, max_streams=8, max_windows_per_stream=3, max_latency=2.0)
    got2 = drive(plain, audio, plan, 5, resume=(8, 0))
    galleries[4] = galleries[5] = None
    check_run(got2, base, plan, galleries, config, seeded)
    for rec, rec2 in zip(got, got2):
        for k in (0, 1, 2, 3):
            if k in rec:
                assert rec[k][0] == rec2[k][0]


def test_one_gallery_per_open_equals_the_default(states, cuda_device):
    config = make_config(states, cuda_device, latency=1.0)
    seeds = [4201, 4202, 4203]
    audio = {k: synth.synth_audio(S + HOP * 16, seed=s) for k, s in enumerate(seeds)}
    rng = np.random.default_rng(3)
    entries, names = [], []
    for k, s in enumerate(seeds):
        p = learned(config, s, [f"q{k}a", f"q{k}b"])
        entries += list(p.centroids)
        names += list(p.names)
    names, table = hidden((names, np.stack(entries)), rng.standard_normal((3000, len(entries[0]))), rng)
    gallery = SpeakerGallery(KnownSpeakers(names, table), 0.3, cuda_device)
    la, lb = [], []
    a = drive(MultiStreamDiarization(config, 4, 3, gallery=gallery), audio, [{}] * 3, 7, launches=la)
    b = drive(MultiStreamDiarization(config, 4, 3), audio, [dict(gallery=gallery)] * 3, 7, launches=lb)
    assert la == lb
    assert [{k: v[0] for k, v in r.items()} for r in a] == [{k: v[0] for k, v in r.items()} for r in b]


def test_a_stream_alone_equals_it_among_300_over_40_galleries(states, cuda_device):
    config = make_config(states, cuda_device, latency=1.0)
    rng = np.random.default_rng(17)
    n, ticks = 300, 10
    p0 = learned(config, 4301, ["zoe", "yan"])
    D = p0.dimension
    names, table = hidden((p0.names, p0.centroids), rng.standard_normal((2000, D)), rng)
    mine = SpeakerGallery(KnownSpeakers(names, table), 1.0, cuda_device)   # generous: the stream's speakers get names
    others = [SpeakerGallery(KnownSpeakers([f"g{j}e{i}" for i in range(G)], rng.standard_normal((G, D))),
                             float(rng.uniform(0.2, 0.6)), cuda_device)
              for j, G in enumerate(rng.choice([16, 700, 3000, 9000], 39))]
    audio0 = synth.synth_audio(S + HOP * (ticks - 1), seed=4302)
    audios = [audio0] + [synth.synth_audio(S + HOP * (ticks - 1), seed=5000 + i) for i in range(n - 1)]

    def run(server, streams, launches):
        sids = [server.open(gallery=g) for g in streams]
        out = []
        for t in range(ticks):
            for sid, a in zip(sids, audios):
                server.push(sid, a[t * HOP:S + t * HOP] if t == 0 else a[S + (t - 1) * HOP:S + t * HOP])
            before = _lib.lib().dg_launch_count()
            server.step()
            launches.append(_lib.lib().dg_launch_count() - before)
            st = server.speakers(sids[0])
            out.append((list(st.names), st.centroids))
        return out

    la, lm, l1 = [], [], []
    alone = run(MultiStreamDiarization(config, 1, 1), [mine], la)
    many = run(MultiStreamDiarization(config, n, 1), [mine] + [others[i % 39] for i in range(n - 1)], lm)
    one = run(MultiStreamDiarization(config, n, 1), [mine] * n, l1)
    for t, ((names_a, c_a), (names_m, c_m)) in enumerate(zip(alone, many)):
        assert np.array_equal(c_a.view(np.int64), c_m.view(np.int64)), f"tick {t}: the centroids differ"
        assert names_a == names_m, f"tick {t}"
    assert lm == l1, (lm, l1)
    assert any(not label.startswith("speaker") for label in alone[-1][0]), alone[-1][0]


def test_refusals_leave_the_slot_closed_and_launch_nothing(states, cuda_device):
    config = make_config(states, cuda_device)
    server = MultiStreamDiarization(config, max_streams=2, max_windows_per_stream=2)
    D = server.D
    lib = _lib.lib()
    rng = np.random.default_rng(1)
    good = SpeakerGallery(KnownSpeakers(["a", "b"], rng.standard_normal((2, D))), 0.5, cuda_device)
    good.handle   # uploaded before counting
    before = lib.dg_launch_count()
    bad = [SpeakerGallery(KnownSpeakers(["a"], np.ones((1, 16))), 0.5, cuda_device),     # another dimension
           SpeakerGallery(KnownSpeakers(["a"], np.ones((1, D))), 0.5, "cpu")]            # another device
    for g in bad:
        with pytest.raises(ValueError):
            server.open(gallery=g)
        assert not server._open.any()
    euclid_cfg = make_config(states, cuda_device)
    euclid_cfg.metric = "euclidean"
    euclid = MultiStreamDiarization(euclid_cfg, 2, 2)
    with pytest.raises(ValueError, match="metric"):
        euclid.open(gallery=good)
    assert not euclid._open.any()
    vad_cfg = blocks.VoiceActivityDetectionConfig(segmentation=config.segmentation, device=cuda_device)
    vad = MultiStreamVoiceActivityDetection(vad_cfg, 2, 2)
    with pytest.raises(ValueError, match="no speakers to name"):
        vad.open(gallery=good)
    assert not vad._open.any()
    assert lib.dg_launch_count() == before
    # the C entry point refuses a VAD handle and a slot after its first tick
    assert lib.dg_multi_set_slot_gallery(vad.handle, 0, good.handle, 0.5) == -1
    sid = server.open(gallery=good)
    assert sid == 0
    server.step()                      # a tick without windows launches nothing
    assert lib.dg_launch_count() == before
    server.push(sid, synth.synth_audio(S, seed=3))
    server.step()
    assert lib.dg_multi_set_slot_gallery(server.handle, sid, good.handle, 0.5) == -1
    assert b"first tick" in lib.dg_last_error()
    torch.cuda.synchronize()


def test_a_query_past_2_31_elements_equals_its_halves(cuda_device):
    """dg_gallery_query over Q x D > 2^31 - 1 query elements runs in several launches of whole claim groups; the result
    equals the two halves queried apart, bit for bit, and the float64 distances"""
    D, Q = 1 << 20, 2080                                   # 2 181 038 080 elements, 17.4 GB
    rng = np.random.default_rng(8)
    E = rng.standard_normal((3, D))
    gal = SpeakerGallery(KnownSpeakers(["a", "b", "c"], E), 2.0, cuda_device)
    gen = torch.Generator(device=cuda_device).manual_seed(3)
    x = torch.randn((Q, D), dtype=torch.float64, device=cuda_device, generator=gen)
    x[::7] += torch.from_numpy(E[1]).to(cuda_device)
    group = torch.arange(Q, dtype=torch.int32, device=cuda_device) // 4
    lib, st = _lib.lib(), _lib.stream_ptr(cuda_device)

    def query(lo, hi):
        e = torch.empty(hi - lo, dtype=torch.int32, device=cuda_device)
        d = torch.empty(hi - lo, dtype=torch.float64, device=cuda_device)
        _lib.check(lib.dg_gallery_query(gal.handle, x[lo:hi].data_ptr(), hi - lo, group[lo:hi].data_ptr(), None, 2.0,
                                        e.data_ptr(), d.data_ptr(), st))
        return e, d

    gal.handle                                             # uploaded (its norms launch) before counting
    before = lib.dg_launch_count()
    e_all, d_all = query(0, Q)
    assert lib.dg_launch_count() - before == 4             # two launches of two kernels
    e1, d1 = query(0, Q // 2)
    e2, d2 = query(Q // 2, Q)
    assert torch.equal(e_all, torch.cat([e1, e2])) and torch.equal(d_all.view(torch.int64), torch.cat([d1, d2]).view(torch.int64))
    Et = torch.from_numpy(E).to(cuda_device)
    c = (x @ Et.T) / (x.norm(dim=1, keepdim=True) * Et.norm(dim=1)[None, :])
    ref = (1 - c.clamp(-1, 1)).min(dim=1).values
    assert (d_all - ref).abs().max().item() <= 1e-12
    del x
    torch.cuda.empty_cache()
