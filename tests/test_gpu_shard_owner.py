"""-m gpu: the owner grouping of the sharded path (merge.cu seed_owner_kernel behind
lib.records_group_by_owner and lib.seeds_group_by_owner) on crafted device records, against a numpy
restatement: the owner of every record's field, the bincount of the owners and its exclusive scan.
  * bounds equal the numpy bounds exactly;
  * group w, rows [bounds[w], bounds[w+1]), holds exactly the input records owned by w (order inside a
    group is free, so the rows are compared sorted) -- nothing is lost or duplicated;
  * a field value at or above the owner map's length (nrc) belongs to rank 0.
The kernel counts and places records in tiles of 2048 per CTA; n runs across those tiles, the world across
1..64 ranks, the seed's icont field below, across, at and above bit 64, with random bits everywhere else."""
import numpy as np
import pytest
import torch

from fastga_b200 import lib, shard

pytestmark = pytest.mark.gpu

TILE = 2048                          # records per CTA of seed_owner_kernel (256 threads x 8)
NS = [0, 1, TILE - 1, TILE, TILE + 1, 3 * TILE - 1, 3 * TILE + 1, 3_000_017]
WORLDS = [1, 2, 3, 7, 8, 63, 64]


def field_of(recs, pos, nbits):
    """the nbits-bit field at bit pos of (n,2) uint64 records [lo, hi] (128-bit little-endian)"""
    lo, hi = recs[:, 0], recs[:, 1]
    if pos >= 64:
        v = hi >> np.uint64(pos - 64)
    elif pos == 0:
        v = lo
    else:
        v = (lo >> np.uint64(pos)) | (hi << np.uint64(64 - pos))
    return (v & np.uint64((1 << nbits) - 1)).astype(np.int64)


def set_field(recs, pos, nbits, vals):
    """writes vals into the nbits-bit field at bit pos, leaving every other bit as it is"""
    mask = ((1 << nbits) - 1) << pos
    lo_m, hi_m = np.uint64(mask & ((1 << 64) - 1)), np.uint64(mask >> 64)
    v = np.asarray(vals, dtype=np.uint64)
    recs[:, 0] &= ~lo_m
    recs[:, 1] &= ~hi_m
    if pos >= 64:
        recs[:, 1] |= (v << np.uint64(pos - 64)) & hi_m
    else:
        recs[:, 0] |= (v << np.uint64(pos)) & lo_m
        if pos + nbits > 64:
            recs[:, 1] |= (v >> np.uint64(64 - pos)) & hi_m


def want_bounds(owners, world):
    return np.concatenate([[0], np.cumsum(np.bincount(owners, minlength=world))]).astype(np.int64)


def run_grouping(recs, call):
    """recs to the device, call(src_ptr, n, dst_ptr) -> bounds; returns (bounds, grouped rows on the host)"""
    n = len(recs)
    src = torch.from_numpy(recs.view(np.int64)).cuda() if n else torch.empty((1, 2), dtype=torch.int64,
                                                                              device="cuda")
    dst = torch.full((max(n, 1), 2), -1, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    bounds = call(src.data_ptr() if n else 0, n, dst.data_ptr())
    return bounds, dst[:n].cpu().numpy().view(np.uint64)


def assert_grouped(recs, owners, world, bounds, got):
    wb = want_bounds(owners, world)
    assert np.array_equal(bounds, wb), (bounds.tolist(), wb.tolist())
    # group of every output row from the bounds; (group, lo, hi) sorted on both sides: each group holds the
    # multiset of its input records, so the output is a permutation of the input
    gw = np.repeat(np.arange(world), np.diff(bounds))
    o_want = np.lexsort((recs[:, 1], recs[:, 0], owners))
    o_got = np.lexsort((got[:, 1], got[:, 0], gw))
    assert np.array_equal(got[o_got], recs[o_want])


def random_records(rng, n):
    return rng.integers(0, 1 << 64, size=(n, 2), dtype=np.uint64, endpoint=False)


def owner256_of(world):
    cuts = shard.top_byte_cuts(world)
    own = np.zeros(256, dtype=np.int32)
    for r in range(world):
        own[cuts[r]:cuts[r + 1]] = r
    return own


def group_records(recs, owner256, world):
    return run_grouping(recs, lambda s, n, d: lib.records_group_by_owner(s, n, owner256, world, d))


def group_seeds(recs, bits, owner, world):
    return run_grouping(recs, lambda s, n, d: lib.seeds_group_by_owner(s, n, bits, owner, world, d))


# ---- k-mer records: owner of the top byte (bits 120..127) ----

@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("n", NS)
def test_records_by_top_byte_cuts(n, world):
    """the owner256 map align_sharded builds from top_byte_cuts(world)"""
    rng = np.random.default_rng(1000 * world + n % 1000)
    recs = random_records(rng, n)
    own = owner256_of(world)
    bounds, got = group_records(recs, own, world)
    assert_grouped(recs, own[field_of(recs, 120, 8)], world, bounds, got)


@pytest.mark.parametrize("world", [2, 3, 8, 64])
@pytest.mark.parametrize("kind", ["one_rank", "interleaved", "idle_ranks"])
def test_records_by_crafted_owner_maps(kind, world):
    """every record to the last rank (each CTA adds 2048 to one counter); owners alternating record by
    record; only every third rank owning anything"""
    rng = np.random.default_rng(world)
    n = 3 * TILE + 1
    recs = random_records(rng, n)
    if kind == "one_rank":
        own = np.full(256, world - 1, dtype=np.int32)
    elif kind == "interleaved":
        own = (np.arange(256) % world).astype(np.int32)
        set_field(recs, 120, 8, np.arange(n) % (256 - 256 % world))
    else:
        own = (3 * rng.integers(0, (world + 2) // 3, 256)).astype(np.int32)
    bounds, got = group_records(recs, own, world)
    owners = own[field_of(recs, 120, 8)]
    if kind == "interleaved":
        assert (owners[1:] != owners[:-1]).all()
    assert_grouped(recs, owners, world, bounds, got)


# ---- seed records: owner of the icont field at bit p_ic = 12 + anti + band + jc ----

#  (p_ic, ic_bits): wholly below bit 64, ending at bit 64, across it (by one bit and by several), starting
#  at it, above it, and up to bit 128
FIELDS = [(15, 1), (20, 5), (49, 15), (57, 7), (60, 8), (63, 2), (58, 13), (64, 1), (64, 15), (70, 3),
          (100, 12), (113, 15)]


def bits_for(p_ic, ic_bits):
    """(anti, band, jc, ic) whose icont field starts at p_ic"""
    jc = 1 + (p_ic - 12) % 3 if p_ic - 12 >= 3 else 1
    band = 1
    return (p_ic - 12 - jc - band, band, jc, ic_bits)


def owner_map(rng, kind, nrc, world):
    if kind == "one_rank":
        return np.full(nrc, world - 1, dtype=np.int32)
    if kind == "interleaved":
        return (np.arange(nrc) % world).astype(np.int32)
    # ranks 1, 4, 7, ... own nothing
    ranks = np.array([r for r in range(world) if r % 3 != 1] or [0])
    return ranks[rng.integers(0, len(ranks), nrc)].astype(np.int32)


def nrc_for(ic_bits):
    """below 2^ic_bits, so that some field values have no owner entry"""
    return max(1, (3 << ic_bits) // 4)


@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("p_ic,ic_bits", FIELDS)
def test_seeds_by_icont_field(p_ic, ic_bits, world):
    rng = np.random.default_rng(p_ic * 100 + ic_bits + world)
    bits = bits_for(p_ic, ic_bits)
    assert 12 + bits[0] + bits[1] + bits[2] == p_ic and min(bits) >= 1
    n = 3 * TILE + 1
    recs = random_records(rng, n)
    nrc = nrc_for(ic_bits)
    own = owner_map(rng, "idle_ranks", nrc, world)
    ic = field_of(recs, p_ic, ic_bits)
    owners = np.where(ic < nrc, own[np.minimum(ic, nrc - 1)], 0)
    bounds, got = group_seeds(recs, bits, own, world)
    assert_grouped(recs, owners, world, bounds, got)


@pytest.mark.parametrize("kind", ["one_rank", "interleaved", "idle_ranks"])
@pytest.mark.parametrize("n", NS)
def test_seeds_at_tile_edges(n, kind):
    """a field straddling bit 64 (p_ic 60, 8 bits), world 7, under the three owner-map shapes"""
    world, p_ic, ic_bits = 7, 60, 8
    rng = np.random.default_rng(n % 7919)
    recs = random_records(rng, n)
    nrc = 1 << ic_bits
    own = owner_map(rng, kind, nrc, world)
    if kind == "interleaved":
        set_field(recs, p_ic, ic_bits, np.arange(n) % nrc)
    ic = field_of(recs, p_ic, ic_bits)
    if kind == "interleaved":
        assert np.array_equal(ic, np.arange(n) % nrc)
    bounds, got = group_seeds(recs, bits_for(p_ic, ic_bits), own, world)
    assert_grouped(recs, own[ic], world, bounds, got)


@pytest.mark.parametrize("p_ic,ic_bits", [(20, 5), (60, 8), (64, 15), (113, 15)])
def test_field_values_without_an_owner_go_to_rank_0(p_ic, ic_bits):
    """icont >= nrc: rank 0, whatever the map says -- here no rank-0 entry at all"""
    world, n = 5, 3 * TILE + 1
    rng = np.random.default_rng(p_ic)
    recs = random_records(rng, n)
    nrc = nrc_for(ic_bits)
    vals = rng.integers(0, 1 << ic_bits, n)
    vals[::3] = rng.integers(nrc, 1 << ic_bits, len(vals[::3]))
    set_field(recs, p_ic, ic_bits, vals)
    assert np.array_equal(field_of(recs, p_ic, ic_bits), vals)
    own = (1 + np.arange(nrc) % (world - 1)).astype(np.int32)
    bounds, got = group_seeds(recs, bits_for(p_ic, ic_bits), own, world)
    owners = np.where(vals < nrc, own[np.minimum(vals, nrc - 1)], 0)
    assert bounds[1] == (vals >= nrc).sum() > 0
    assert_grouped(recs, owners, world, bounds, got)


@pytest.mark.parametrize("world", [0, 65])
def test_world_outside_1_to_64_is_refused(world):
    recs = random_records(np.random.default_rng(1), 10)
    with pytest.raises(lib.FgbError):
        group_records(recs, np.zeros(256, dtype=np.int32), world)
    with pytest.raises(lib.FgbError):
        group_seeds(recs, bits_for(60, 8), np.zeros(256, dtype=np.int32), world)


@pytest.mark.parametrize("bad", [-1, 3])
def test_owner_outside_the_world_is_refused(bad):
    """an owner map entry that names no rank of the world (here world 3)"""
    recs = random_records(np.random.default_rng(2), 10)
    own = np.zeros(256, dtype=np.int32)
    own[200] = bad
    with pytest.raises(lib.FgbError):
        group_records(recs, own, 3)
    with pytest.raises(lib.FgbError):
        group_seeds(recs, bits_for(60, 8), own, 3)
