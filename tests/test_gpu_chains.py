"""-m gpu: chain detection, the stage between the seed sort and the extension (band segments, prefilter,
chain_plan / chain_chunk / chain_stitch), read out on its own by lib.chain_hits and compared with the
oracle's chain scan (oracle_lib.chains) on the same seed records: the work triples, and the hit list of
every long triple entry by entry, at chunk sizes from one seed to one chunk per triple.  Then the extension
at chunk sizes that cut elsewhere, and without chain detection: the same records every time."""
import os

import numpy as np
import pytest

import edge_cases
import oracle_lib as ol
import param_cases as pc
from fastga_b200 import formats, lib, synth
from test_gpu_stages import _canon
from test_oracle_pin import _self_genomes

pytestmark = pytest.mark.gpu

DEFAULT_CHUNK = 1536                     # merged seeds per chunk of fgb_extend
HCAP = 48                                # hits a chunk records; a chunk with more sends its triple to the kernel
CHUNKOUT_BYTES = 1240                    # device bytes per chunk (struct ChunkOut)
CHUNKS = [1, 2, 3, 31, 32, 33, 80, 81, 97, DEFAULT_CHUNK, 1 << 30]
LISTLESS = lib.CHAIN_LISTLESS


def _pair(name):
    """(A contigs, B contigs or None for SELF, chain parameters) of a case"""
    if name == "small_pair":
        A, B = synth.make_pair(11, 1_200_000, 3, 0.05, sv_every=60000)
        return A, B, {}
    if name in pc.CASES:
        flags, A, B = pc.case(name)
        p = pc.params(flags)
        return A, B, {k: p[k] for k in ("chain_break", "chain_min") if k in p}
    if name == "self_tandem61":
        return _self_genomes()["tandem61"], None, {}
    A, B, _, _ = edge_cases.CASES[name]()
    return A, B, {}


class Staged:
    """device genomes and seeds of a case, and the seed records they hold"""

    def __init__(self, name):
        A, B, self.chain = _pair(name)
        self.gA = formats.genome_from_arrays(A)
        self.gB = self.gA if B is None else formats.genome_from_arrays(B)
        self.dA = lib.DeviceGenome(self.gA, want_revcomp=True)
        self.dB = self.dA if B is None else lib.DeviceGenome(self.gB)
        xA = lib.DeviceGix.build(self.dA)
        amx, bmx = int(self.gA.clen.max()), int(self.gB.clen.max())
        if B is None:
            self.seeds = lib.DeviceSeeds.find_self(xA, amx, 10)
        else:
            xB = lib.DeviceGix.build(self.dB)
            self.seeds = lib.DeviceSeeds.find(xA, xB, amx, bmx, 10)
            xB.close()
        xA.close()
        self.recs = self.seeds.download()
        self.layout = self.seeds.layout + (amx, bmx)
        self.self_mode = B is None

    def close(self):
        for h in (self.seeds, self.dA, self.dB):
            h.close()


@pytest.fixture(scope="module")
def staged():
    """case name -> Staged, one case held at a time"""
    cache = {}

    def get(name):
        if name not in cache:
            for s in cache.values():
                s.close()
            cache.clear()
            cache[name] = Staged(name)
        return cache[name]
    yield get
    for s in cache.values():
        s.close()


def _check_run(S, otr, oh, chunk, trip, hits, info):
    """one chain_hits run against the oracle's triples otr and chains oh; returns the chunks per long triple"""
    cb, cm = S.chain.get("chain_break", 2000), S.chain.get("chain_min", 170)
    osize = otr["e"] - otr["b"]
    at = {int(b): q for q, b in enumerate(otr["b"])}
    # the work triples are scanned triples of the oracle, each once, with the oracle's extent
    assert len(trip) == info["work"] > 0
    assert all(int(s) in at for s in trip["start"])
    k = np.array([at[int(s)] for s in trip["start"]])
    assert len(set(k.tolist())) == len(k)
    assert np.array_equal(trip["end"], otr["e"][k])
    size = trip["end"] - trip["start"]
    long_ = trip["long"] == 1
    assert np.array_equal(long_, size > 64)
    assert long_[:info["long"]].all() and not long_[info["long"]:].any()
    # long ones first, largest first
    assert (np.diff(size[:info["long"]]) <= 0).all()
    # what the prefilter dropped: too few seeds for chain_min, or at most 64 seeds and no chain
    dropped = np.ones(len(otr), bool)
    dropped[k] = False
    assert ((osize[dropped] < (cm + 79) // 80) | ((osize[dropped] <= 64) & (otr["nh"][dropped] == 0))).all()
    assert (otr["nh"][osize < (cm + 79) // 80] == 0).all()
    # a short work triple holds a chain
    assert (otr["nh"][k[~long_]] > 0).all()

    listless = (trip["hn"] & LISTLESS) != 0
    assert listless[~long_].all() and (trip["key"][~long_] == -1).all()
    if chunk == 0:
        assert listless.all() and info["chunks"] == 0
        return np.zeros(0, np.int64)
    # the capacity of the hit slots was not what took a list away
    assert info["reserved"] <= info["capacity"]
    nch = np.maximum((size[long_] + chunk - 1) // chunk, 1)
    assert info["chunks"] == int(nch.sum())
    kl = k[long_]
    assert np.array_equal(trip["key"][long_], otr["key"][kl])
    assert np.array_equal(trip["band"][long_], otr["cdiag"][kl])
    fields = ("alow", "ahgh", "dgmin", "dgmax")
    for w in np.nonzero(long_)[0]:
        o = otr[k[w]]
        want = oh[o["h0"]:o["h0"] + o["nh"]]
        if listless[w]:
            # only a chunk with more than 48 chains takes the list away
            assert o["nh"] > HCAP, (chunk, int(trip["start"][w]), int(o["nh"]))
            continue
        h0, hn = int(trip["h0"][w]), int(trip["hn"][w])
        got = hits[h0:h0 + hn]
        assert hn == len(want), (chunk, int(trip["start"][w]), hn, len(want))
        for f in fields:
            assert np.array_equal(got[f], want[f]), (chunk, int(trip["start"][w]), f)
    return nch


CASES = ["small_pair", "short_chains", "long_break", "tandem_repeats", "identical_and_revcomp", "long_contigs",
         "self_tandem61", "chain_islands"]


@pytest.mark.parametrize("name", CASES)
def test_chain_lists_match_oracle_at_every_chunk_size(name, staged):
    S = staged(name)
    cb, cm = S.chain.get("chain_break", 2000), S.chain.get("chain_min", 170)
    # the look-back at a chunk cut and the prefilter's seed bound both take a seed to cover <= 80 anti-diagonals
    assert int((S.recs[:, 0] & np.uint64(63)).max()) <= 40
    otr, oh = ol.chains(S.recs, S.layout, cb, cm)
    assert len(oh) > 0
    base = lib.device_live_bytes()
    trip, _, info = lib.chain_hits(S.seeds, cb, cm, chunk=0)
    _check_run(S, otr, oh, 0, trip, np.zeros(0, lib.CHAIN_HIT_DT), info)
    lsize = (trip["end"] - trip["start"])[trip["long"] == 1]
    assert len(lsize) > 0
    ran = []
    for chunk in CHUNKS:
        nplan = int(np.maximum((lsize + chunk - 1) // chunk, 1).sum())
        if nplan * CHUNKOUT_BYTES > 1 << 30:
            continue
        trip, hits, info = lib.chain_hits(S.seeds, cb, cm, chunk=chunk)
        nch = _check_run(S, otr, oh, chunk, trip, hits, info)
        assert lib.device_live_bytes() == base
        listless = (trip["long"] == 1) & ((trip["hn"] & LISTLESS) != 0)
        # the regime of the run: cuts inside the triples, or none
        if chunk == 1 << 30:
            assert nch.max() == 1
        elif chunk <= 97:
            assert nch.max() >= 10
        if chunk <= 33:
            # some chain spans ten chunks or more (merged seeds of a chain are consecutive)
            kl = np.array([np.searchsorted(otr["b"], s) for s in trip["start"][trip["long"] == 1]])
            spans = [oh[otr["h0"][q]:otr["h0"][q] + otr["nh"][q]]["nseed"].max(initial=0) for q in kl]
            assert max(spans) > 10 * chunk
        if chunk == DEFAULT_CHUNK and edge_cases.REGIMES.get(name, {}).get("chunk_overflow"):
            assert listless.any()
        ran.append(chunk)
    assert DEFAULT_CHUNK in ran and 1 << 30 in ran and min(ran) <= 33


def _crafted_seeds():
    """seed records of one band-pair triple (bands 5 and 6 of one contig pair) built to put chunk cuts where
    they are hard, with chain_break 200 and chain_min 50.  Three times: a seed of lcp 40 (it reaches 80
    anti-diagonals past its own), 32 seeds of lcp 1 two anti-diagonals apart that start 10 past it and
    never reach as far, then, past chain_break, a seed that closes the chain.  At a cut before that seed the
    running maximum sits 62 anti-diagonals and 32 seeds back in its band.  Then 40 pairs of seeds on equal
    anti-diagonals in the two bands, three apart, where cuts fall between the two of a pair."""
    band, lcp, dg, anti = [], [], [], []
    for base in (1_000, 2_000, 3_000):
        for a, l in [(base, 40)] + [(base + 10 + 2 * i, 1) for i in range(32)] + [(base + 300, 20)]:
            band.append(5); lcp.append(l); dg.append(1); anti.append(a)
    for i in range(40):
        for b in (5, 6):
            band.append(b); lcp.append(8 + (i * 7 + b) % 30); dg.append(2 * b); anti.append(5_000 + 3 * i)
    bits = (20, 14, 1, 1)
    rec = np.zeros((len(band), 2), dtype=np.uint64)
    rec[:, 0] = (np.array(lcp, np.uint64) | (np.array(dg, np.uint64) << np.uint64(6)) |
                 (np.array(anti, np.uint64) << np.uint64(12)) | (np.array(band, np.uint64) << np.uint64(12 + bits[0])))
    return rec, bits


def test_chain_lists_match_oracle_at_crafted_cuts():
    """the look-back that rebuilds the running maximum at a cut must reach 80 anti-diagonals back, past the
    32 seeds it reads at a time; a cut between seeds of equal anti-diagonal in the two bands"""
    import torch
    from types import SimpleNamespace
    rec, bits = _crafted_seeds()
    d = torch.from_numpy(rec.view(np.int64).copy()).cuda()
    torch.cuda.synchronize()
    amx = bmx = 1 << 18
    seeds = lib.seeds_from_records(d.data_ptr(), len(rec), bits, amx, bmx)
    del d
    S = SimpleNamespace(chain=dict(chain_break=200, chain_min=50), recs=seeds.download())
    layout = bits + (amx, bmx)
    otr, oh = ol.chains(S.recs, layout, 200, 50)
    assert len(otr) == 1 and list(oh["ahgh"][:3]) == [1_080, 2_080, 3_080] and len(oh) == 4
    for chunk in (1, 2, 3, 33, DEFAULT_CHUNK):
        trip, hits, info = lib.chain_hits(seeds, 200, 50, chunk=chunk)
        _check_run(S, otr, oh, chunk, trip, hits, info)
        assert info["long"] == 1 and (trip["hn"][0] & LISTLESS) == 0
    seeds.close()


COUNTS = ("hits", "la_calls")


def _extend(S, chunk):
    """records (fields but the sequence number, and trace bytes, in discovery order) and work counters of
    fgb_extend with FGB_CHAIN_CHUNK = chunk (None: unset)"""
    old = os.environ.pop("FGB_CHAIN_CHUNK", None)
    if chunk is not None:
        os.environ["FGB_CHAIN_CHUNK"] = chunk
    try:
        ov = lib.DeviceOverlaps.extend(S.seeds, S.dA, S.dB, S.gA.freq, **S.chain)
    finally:
        os.environ.pop("FGB_CHAIN_CHUNK", None)
        if old is not None:
            os.environ["FGB_CHAIN_CHUNK"] = old
    try:
        recs, pool = ov.records()
        cnt = ov.counters()
    finally:
        ov.close()
    fields = [n for n in recs.dtype.names if n not in ("toff", "seq")]
    out = [tuple(int(r[n]) for n in fields) + (pool[r["toff"]:r["toff"] + r["tlen"]].tobytes(),) for r in recs]
    return out, {k: cnt[k] for k in COUNTS}, recs, pool


@pytest.mark.parametrize("name", ["short_chains", "tandem_repeats", "chain_islands"])
def test_extension_is_the_same_at_any_chunk_size_and_without_chain_detection(name, staged):
    """FGB_CHAIN_CHUNK unset, 3, 33 and 0 (no chain detection: every triple is scanned in the kernel, and
    the first launch is not a hit-group launch): the same records and counts, and the oracle's"""
    S = staged(name)
    want, wcnt, recs, pool = _extend(S, None)
    for chunk in ("3", "33", "0"):
        got, gcnt, _, _ = _extend(S, chunk)
        assert got == want, chunk
        assert gcnt["hits"] == wcnt["hits"], chunk
        if chunk == "0":
            # la_calls counts every Local_Alignment call run: with hit lists, those of hit groups that
            # start with a clear tube and of the triples re-run when a group reached the next one, whose
            # records are dropped; a triple scanned in one piece runs only the calls of the result
            assert gcnt["la_calls"] <= wcnt["la_calls"]
        else:
            assert gcnt["la_calls"] == wcnt["la_calls"], chunk
    ov, tp, nhit = ol.search(S.recs, S.layout, S.gA, S.gB, S.dA.perm, S.dB.perm, S.gA.freq, **S.chain)
    assert wcnt["hits"] == nhit
    jb, ib = S.layout[2], S.layout[3]
    pk = recs["pairkey"].astype(np.int64)
    jc, ic, comp = pk & ((1 << jb) - 1), (pk >> jb) & ((1 << ib) - 1), pk >> (jb + ib)
    g = _canon(recs, pool, S.dA.perm[ic], S.dB.perm[jc], comp)
    assert len(g) > 20 and g == _canon(ov, tp)
