"""-m gpu: the seed stage on the crafted seed records of seed_stage_cases.py.  Each case is sorted from bit 6
(lib.seeds_from_records) and read out by lib.chain_hits at chunk sizes 1, 33 and 1536, with the long-triple
sort cap (FGB_LONG_SORT_CAP) unset, 0, one below the case's long count and at it: the band segments, every
work triple's [start, end), the long triples in launch order (or, unsorted, as a set), the short work
triples as a set, the chunk plan and every long triple's hit list, against the numpy restatement and the
oracle's chain scan.  The cases with genomes then go through fgb_extend and fgb_filter -- default, without
chain detection and under each cap -- and must give the oracle's records, trace bytes and hit count."""
import os

import numpy as np
import pytest

import oracle_lib as ol
import seed_stage_cases as sc
from fastga_b200 import formats, lib
from test_gpu_seed_stage import _numpy_triples

pytestmark = pytest.mark.gpu

HCAP = 48                       # hits a chunk records
CHUNKS = (1, 33, 1536)
CHUNKOUT_BYTES = 1240           # device bytes per chunk (struct ChunkOut)
PLAN_BUDGET = 2 << 30           # chunk sizes whose plan needs more are skipped
KNOBS = ("FGB_LONG_SORT_CAP", "FGB_CHAIN_CHUNK")
LISTLESS = lib.CHAIN_LISTLESS


def _env(env):
    for k in KNOBS:
        os.environ.pop(k, None)
    os.environ.update(env)


@pytest.fixture
def knobs():
    yield _env
    _env({})


def _upload(C):
    import torch
    d = torch.from_numpy(C.recs.view(np.int64).copy()).cuda()
    torch.cuda.synchronize()
    s = lib.seeds_from_records(d.data_ptr(), len(C.recs), C.layout[:4], C.layout[4], C.layout[5])
    del d
    return s


def _caps(F):
    """(env, sorted) of each sort cap a case runs under: unset, 0, nlong - 1, nlong"""
    out = [({}, F.nlong <= sc.LONG_SORT_CAP)]
    for cap in sorted({0, F.nlong - 1, F.nlong}):
        if cap >= 0:
            out.append(({"FGB_LONG_SORT_CAP": str(cap)}, F.nlong <= cap))
    return out


def _check_triples(C, F, trip, hits, info, chunk, sorted_):
    nl = F.nlong
    assert info["work"] == len(trip) == nl + len(F.short_work)
    start = trip["start"]
    q = np.searchsorted(F.seg, start)
    assert (q < len(F.seg)).all() and np.array_equal(F.seg[q], start)
    assert np.array_equal(F.e[q], trip["end"])
    assert len(np.unique(start)) == len(start)
    assert set(start[:nl].tolist()) == {int(F.seg[j]) for j in F.lj}
    assert set(start[nl:].tolist()) == F.short_work
    if not sorted_:
        # past the cap: no sort and no chain detection; every triple is scanned in the kernel
        assert info["long"] == 0 and info["chunks"] == 0 and info["slots"] == 0
        assert not trip["long"].any() and ((trip["hn"] & LISTLESS) != 0).all()
        return
    assert info["long"] == nl
    assert np.array_equal(start[:nl], F.seg[F.lj]) and np.array_equal(trip["end"][:nl], F.e[F.lj])
    assert (trip["long"][:nl] == 1).all() and not trip["long"][nl:].any()
    assert ((trip["hn"][nl:] & LISTLESS) != 0).all()
    if nl == 0:
        assert info["chunks"] == 0
        return
    size = F.size[F.lj]
    nch = np.maximum((size + chunk - 1) // chunk, 1)
    assert info["chunks"] == int(nch.sum())
    assert info["capacity"] == int(nch.sum()) * (HCAP + 1) + info["work"] + 16
    k = np.searchsorted(F.otr["b"], start[:nl])
    nh = F.otr["nh"][k]
    hn = trip["hn"][:nl].astype(np.int64)
    listless = (hn & LISTLESS) != 0
    assert (nh[listless] > HCAP).all()
    assert np.array_equal(hn[~listless], nh[~listless])
    for w in np.nonzero(~listless & (nh > 0))[0]:
        o = F.otr[k[w]]
        want = F.oh[o["h0"]:o["h0"] + o["nh"]]
        got = hits[trip["h0"][w]:trip["h0"][w] + hn[w]]
        for f in ("alow", "ahgh", "dgmin", "dgmax"):
            assert np.array_equal(got[f], want[f]), (chunk, int(start[w]), f)


class Genomes:
    def __init__(self, A, B):
        self.gA, self.gB = formats.genome_from_arrays(A), formats.genome_from_arrays(B)
        self.dA, self.dB = lib.DeviceGenome(self.gA, want_revcomp=True), lib.DeviceGenome(self.gB)

    def close(self):
        self.dA.close()
        self.dB.close()


def _dummy():
    """contigs the extension never reads: every triple is below the seed bound of chain_min 2^30"""
    rng = np.random.default_rng(1)
    return Genomes([rng.integers(0, 4, 100 + c, dtype=np.uint8) for c in range(4)],
                   [rng.integers(0, 4, 200 + c, dtype=np.uint8) for c in range(4)])


def _extend(C, S, G, chain_min=None):
    """fgb_extend and fgb_filter: (records as the oracle gives them, with trace bytes; counters; filtered)"""
    ov = lib.DeviceOverlaps.extend(S, G.dA, G.dB, G.gA.freq, chain_break=C.chain_break,
                                   chain_min=C.chain_min if chain_min is None else chain_min)
    try:
        recs, pool = ov.records()
        cnt = ov.counters()
        alns = lib.filter_overlaps(ov.h, G.dA.perm, G.dB.perm, C.layout[2], C.layout[3])
    finally:
        ov.close()
    jb, ib = C.layout[2], C.layout[3]
    rows = []
    for r in recs:
        pk = int(r["pairkey"])
        rows.append((pk >> (jb + ib), int(G.dA.perm[(pk >> jb) & ((1 << ib) - 1)]), int(G.dB.perm[pk & ((1 << jb) - 1)]),
                     int(r["abpos"]), int(r["bbpos"]), int(r["aepos"]), int(r["bepos"]), int(r["diffs"]),
                     pool[r["toff"]:r["toff"] + r["tlen"]].tobytes()))
    return rows, cnt, alns


@pytest.mark.parametrize("name", sc.NAMES)
def test_seed_stage_matches_oracle_on_crafted_records(name, knobs):
    C = sc.case(name)
    F = C.facts
    S = _upload(C)
    G = Genomes(*C.genomes) if C.genomes is not None else _dummy()
    try:
        assert S.n == F.n and np.array_equal(S.download(), C.recs)
        if F.n:
            seg, e, kept = _numpy_triples(C.recs, C.layout, C.chain_min)
            assert np.array_equal(seg, F.seg) and np.array_equal(e[kept], F.e[F.kept])
        ran = []
        for env, sorted_ in _caps(F):
            for chunk in (CHUNKS if sorted_ else (1536,)):
                nplan = int(np.maximum((F.size[F.lj] + chunk - 1) // chunk, 1).sum())
                if nplan * CHUNKOUT_BYTES > PLAN_BUDGET:
                    continue
                knobs(env)
                trip, hits, info = lib.chain_hits(S, C.chain_break, C.chain_min, chunk=chunk)
                knobs({})
                _check_triples(C, F, trip, hits, info, chunk, sorted_)
                ran.append((sorted_, chunk))
        assert (True, 1536) in ran and (F.nlong == 0 or (False, 1536) in ran), ran
        if C.genomes is None:
            # the band segments fgb_extend counts, with every triple below the seed bound
            _, cnt, _ = _extend(C, S, G, chain_min=1 << 30)
            assert cnt["nseg"] == len(F.seg) and cnt["nwork"] == 0
            return
        want, wpool, whits = ol.search(C.recs, C.layout, G.gA, G.gB, G.dA.perm, G.dB.perm, G.gA.freq,
                                       chain_break=C.chain_break, chain_min=C.chain_min)
        rows = [(int(r["comp"]), int(r["aread"]), int(r["bread"]), int(r["abpos"]), int(r["bbpos"]),
                 int(r["aepos"]), int(r["bepos"]), int(r["diffs"]),
                 bytes(wpool[int(r["toff"]):int(r["toff"]) + int(r["tlen"])])) for r in want]
        walns = ol.filter(want, wpool)
        got = {}
        for label, env in [("default", {}), ("scan", {"FGB_CHAIN_CHUNK": "0"})] + \
                [("cap%d" % int(e["FGB_LONG_SORT_CAP"]), e) for e, _ in _caps(F)[1:]]:
            knobs(env)
            g, cnt, alns = _extend(C, S, G)
            knobs({})
            assert g == rows, label
            assert cnt["hits"] == whits, label
            assert cnt["nseg"] == len(F.seg) and cnt["nwork"] == F.nlong + len(F.short_work), label
            assert ol.alignment_differences(alns, walns) == "", label
            got[label] = g
        if name.startswith("past_2^20"):
            assert len(rows) > 0
            # two runs in the prefilter's atomic order give the same records
            assert got["cap0"] == got["cap%d" % (F.nlong - 1)]
    finally:
        S.close()
        G.close()
