"""CPU: the CTA-pair exchange of `pointnet_pass_kernel<false>` on tests/pass_schedule.py's model of it.

For tile totals 1 ... 70 and 0 ... 12 queries per stream, both warpgroups and three interleavings of the two CTAs of a
cluster (every store landing at once, every store landing as late as possible, a seeded random order):
  - every tile of every query is produced exactly once per pair of CTAs, and enters each CTA's big layer exactly once,
    into the maxima of its own query;
  - the k-th tile a warpgroup sends is the k-th its peer receives, of the same query and the same pair of tiles;
  - every wait's parity is that of the phase in which its store or arrival lands, and the barrier is in the next phase
    when the wait passes; no store lands in a slot before the previous tile was read; no deadlock (run_pair);
  - per stream, the two CTAs produce equally many tiles over every two consecutive queries.
For every split of the tile total into two segments, every produced tile reads the segment and local tile the host's
layout gives it.  The host's stream assignment gives every query of the batch to exactly one stream.
"""
import collections
import functools

import pytest

import pass_schedule as ps

TILE_TOTALS = range(1, 71)
MAX_QUERIES = 12


@functools.lru_cache(maxsize=None)
def _run(tpq, wg, nq, schedule):
    return ps.run_pair(wg, nq, tpq, schedule, seed=tpq * 1000 + nq * 10 + wg)


def _check_pair(tpq, wg, nq, r):
    queries = range(wg, nq, ps.KWG)
    every = {(qi, t): 1 for qi in queries for t in range(tpq)}
    produced = collections.Counter((qi, tq) for p in (0, 1) for qi, _, tq in r['produce'][p])
    assert produced == every, 'tiles produced per pair: %s' % sorted(set(produced.items()) ^ set(every.items()))[:4]
    for p in (0, 1):
        for qi, i, tile in r['big'][p]:
            # the tile belongs to this query and to the pair of the current step
            assert tile[0] == qi and tile[1] >> 1 == i >> 1, (p, qi, i, tile)
        entered = collections.Counter((qi, tile[1]) for qi, _, tile in r['big'][p])
        assert entered == every, 'part %d: tiles into the big layer: %s' % (p, sorted(set(entered.items()) ^ set(every.items()))[:4])
        # the k-th receive is the peer's k-th send, and the tile it sent
        sent = [(qi, tq) for qi, _, tq in r['produce'][p ^ 1]]
        got = r['recv'][p]
        assert [k for k, _ in got] == list(range(len(sent))), p
        assert [tile[:2] for _, tile in got] == sent, p
        nsend, nrecv = r['counts'][p]
        assert nsend == len(r['produce'][p]) and nsend + nrecv == tpq * len(queries)
    waits = r['waits']
    assert all(parity == phase & 1 for _, _, parity, phase in waits)
    assert len(waits) == sum(n for _, n in r['counts'].values()) + sum(max(n - 1, 0) for n, _ in r['counts'].values())


@pytest.mark.parametrize('tpq', TILE_TOTALS)
def test_exchange_schedule(tpq):
    for nq in range(MAX_QUERIES + 1):
        for schedule in ps.SCHEDULES:
            runs = [_run(tpq, wg, nq, schedule) for wg in range(ps.KWG)]
            for wg, r in enumerate(runs):
                _check_pair(tpq, wg, nq, r)
            # per stream: over queries qi < n, part 0 and part 1 produce equally many tiles for even n, at most one apart
            # for odd n (only the lone last tile of an odd total is not split evenly, and its owner alternates)
            made = {p: collections.Counter(qi for r in runs for qi, _, _ in r['produce'][p]) for p in (0, 1)}
            for n in range(nq + 1):
                d = sum(made[0][qi] for qi in range(n)) - sum(made[1][qi] for qi in range(n))
                assert abs(d) <= n % 2, (tpq, nq, schedule, n, d)


@pytest.mark.parametrize('tpq', TILE_TOTALS)
def test_segments_of_two_segment_launches(tpq):
    for s0 in range(1, tpq + 1):
        s1 = tpq - s0
        assert ps.tiles_per_query(s0, s1) == tpq
        layout = [(0, j) for j in range(s0)] + [(1, j) for j in range(s1)]
        for wg in range(ps.KWG):
            r = _run(tpq, wg, MAX_QUERIES, 'stores_land_at_once')
            per_query = collections.defaultdict(list)
            for p in (0, 1):
                for qi, i, tq in r['produce'][p]:
                    seg = ps.segment(i, tq, s0)
                    assert seg == layout[tq], (s0, s1, wg, p, qi, i, tq, seg)
                    per_query[qi].append(seg)
            assert all(sorted(v) == layout for v in per_query.values()), (s0, s1, wg)
            # the boundary falls inside a pair when s0 is odd: then both CTAs produce, over the queries, the last tile of
            # segment 0 and the first of segment 1 of that pair
            if s0 % 2 and s1:
                for p in (0, 1):
                    made = {tq for _, _, tq in r['produce'][p]}
                    assert {s0 - 1, s0} <= made, (s0, s1, wg, p)


def test_segment_sizes():
    assert [ps.seg_tiles(n) for n in (0, 1, 8, 63, 64, 65, 75, 128, 129, 300, 1000, 1200, 1536, 4096)] == \
        [0, 1, 1, 1, 1, 2, 2, 2, 3, 5, 16, 19, 24, 64]


@pytest.mark.parametrize('clusters', [1, 2, 16, 33, 66])
def test_streams_partition_the_batch(clusters):
    for B in list(range(0, 200)) + [8 * clusters - 1, 8 * clusters, 12 * clusters + 1, 8191, 8192]:
        ns = ps.stream_count(B, clusters)
        seen, counts = [], []
        for stream in range(ns):
            nq = ps.queries_of_stream(B, stream, ns)
            counts.append(nq)
            seen += [ps.query_index(stream, qi, ns) for qi in range(nq)]
        assert sorted(seen) == list(range(B)), (clusters, B)
        assert not counts or max(counts) - min(counts) <= 1


def test_mbarrier_phases():
    # full: one arrival plus the slot's bytes; the bytes may land before the arrival that expects them
    b = ps.MBarrier(1)
    b.arrive(1, ps.SLOT_BYTES)
    assert b.phase == 0 and b.passes(1) and not b.passes(0)
    b.complete_tx(ps.SLOT_BYTES, tag='a')
    assert b.phase == 1 and b.landed['a'] == 0 and b.passes(0) and not b.passes(1)
    b.complete_tx(ps.SLOT_BYTES, tag='b')
    assert b.phase == 1 and b.landed['b'] == 1
    b.arrive(1, ps.SLOT_BYTES)
    assert b.phase == 2 and b.passes(1)
    e = ps.MBarrier(128)
    e.arrive(127)
    assert e.phase == 0
    e.arrive(1)
    assert e.phase == 1
    with pytest.raises(ps.ScheduleError):
        e.arrive(129)
