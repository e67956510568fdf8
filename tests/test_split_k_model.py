"""CPU model of the GEMM's stream-K head (deterministic split-K of what would be a partial last wave): a Python transcription
of `next_unit`, `sk_range_lo`, `sk_owner` and of the slab / ticket exchange in cubecl_b200/csrc/gemm_wgmma.cu, checked for
the invariants the kernel relies on -- every (tile, k-block) is computed exactly once, every unit is non-empty, the number of
partial units of a tile equals the `parts` the ticket waits for, the slab a finishing CTA reads for part j is the slab the unit
that computed part j wrote, and the reduced tile does not depend on which part arrives last."""
import itertools
import random

import numpy as np


def sk_range_lo(r, sk_tiles, num_kb, ranges):
    return (r * sk_tiles * num_kb) // ranges


def sk_owner(x, sk_tiles, num_kb, ranges):
    return ((x + 1) * ranges - 1) // (sk_tiles * num_kb)


def units_of_cluster(c, C, full_tiles, sk_tiles, ranges, umax, num_kb):
    """The work-unit sequence of CTA pair c: (tile, kb0, kb1, slab, partial) -- same integer arithmetic as the device iterator."""
    out = []
    r = c
    while sk_tiles and r < ranges:
        pos, hi, u = sk_range_lo(r, sk_tiles, num_kb, ranges), sk_range_lo(r + 1, sk_tiles, num_kb, ranges), 0
        while pos < hi:
            tau = pos // num_kb
            t0 = tau * num_kb
            end = min(hi, t0 + num_kb)
            kb0, kb1 = pos - t0, end - t0
            out.append((full_tiles + tau, kb0, kb1, r * umax + u, not (kb0 == 0 and kb1 == num_kb)))
            pos, u = end, u + 1
        r += C
    t = c
    while t < full_tiles:
        out.append((t, 0, num_kb, 0, False))
        t += C
    return out


def host_plan(tiles, clusters, num_kb, option="auto", eligible=True):
    """capi.cpp sk_plan -> (time, sk_tiles, ranges, umax)."""
    full_waves, rem = divmod(tiles, clusters)
    time = float(full_waves + (1 if rem else 0))
    none = (time, 0, 0, 0)
    if option == "off" or not eligible or rem == 0 or num_kb < 2:
        return none
    total_kb = rem * num_kb

    def model(ranges, even):
        share = -(-total_kb // ranges)
        parts = max(1.0, ranges / rem)
        head = -(-ranges // clusters) * share / num_kb
        overhead = (4.0 if full_waves >= 1 else 14.0 + 8.0 * parts) / num_kb
        return full_waves + (1.4 if even else 1.6) * head + overhead

    force, even = False, True
    if option in ("auto", "on"):
        force = option == "on"
        s_fit = min(clusters // rem, 8)
        if s_fit >= 2:
            best = s_fit
            if full_waves == 0:
                for s2 in range(2, s_fit + 1):
                    if num_kb // s2 >= 8 and model(rem * s2, True) < model(rem * best, True) - 1e-12:
                        best = s2
            ranges = rem * best
        else:
            ranges, even = clusters, False
    else:
        want = int(option)
        if want == 1:
            return none
        ranges, force = rem * want, True
    ranges = min(ranges, total_kb)
    if ranges <= rem and not force:
        return none
    share = -(-total_kb // ranges)
    t_sk = model(ranges, even)
    if not force:
        if share < 8 or t_sk > 0.96 * time:
            return none
    return (t_sk, rem, ranges, -(-share // num_kb) + 1)


def test_units_cover_every_tile_and_k_block_once_and_parts_match_the_tickets():
    rng = random.Random(7)
    for _ in range(400):
        clusters = rng.choice([37, 74, 148])
        total_tiles = rng.randint(1, 600)
        num_kb = rng.randint(2, 400)
        option = rng.choice(["on", "2", "3", "4", "5", "8", "auto"])
        _, sk_tiles, ranges, umax = host_plan(total_tiles, clusters, num_kb, option)
        full_tiles = total_tiles - sk_tiles
        C = min(max(full_tiles, ranges), clusters) if sk_tiles else min(total_tiles, clusters)
        seen, partial_units, slabs = {}, {}, set()
        for c in range(C):
            for (tile, kb0, kb1, slab, partial) in units_of_cluster(c, C, full_tiles, sk_tiles, ranges, umax, num_kb):
                assert 0 <= kb0 < kb1 <= num_kb                          # never an empty unit
                for kb in range(kb0, kb1):
                    assert (tile, kb) not in seen
                    seen[(tile, kb)] = c
                if partial:
                    assert tile >= full_tiles
                    assert slab not in slabs and slab < ranges * umax    # one slab per partial unit, inside the allocation
                    slabs.add(slab)
                    partial_units.setdefault(tile - full_tiles, []).append((kb0, slab))
        assert len(seen) == total_tiles * num_kb                         # nothing skipped, nothing doubled
        for tau, units in partial_units.items():
            first = sk_owner(tau * num_kb, sk_tiles, num_kb, ranges)
            parts = sk_owner((tau + 1) * num_kb - 1, sk_tiles, num_kb, ranges) - first + 1
            assert parts == len(units) >= 2                              # the ticket waits for exactly the units that exist
            units.sort()                                                 # k order
            for j, (_, slab) in enumerate(units):                        # part_slab(j) in the kernel
                r = first + j
                u = tau - sk_range_lo(r, sk_tiles, num_kb, ranges) // num_kb
                assert r * umax + u == slab
        if sk_tiles:
            assert sk_tiles * (2 if clusters <= 74 else 1) <= 1024       # tickets: one per (tile, CTA rank) in a 1024-entry area


def test_head_runs_before_whole_tiles_on_every_pair():
    # the partial tiles go FIRST so that their slab exchange is hidden under the whole tiles that follow
    for tiles, clusters, num_kb in ((256, 74, 128), (128 + 17, 37, 64), (600, 148, 33)):
        _, sk_tiles, ranges, umax = host_plan(tiles, clusters, num_kb, "on")
        assert sk_tiles == tiles % clusters
        full = tiles - sk_tiles
        for c in range(clusters):
            seq = units_of_cluster(c, clusters, full, sk_tiles, ranges, umax, num_kb)
            kinds = [t >= full for (t, *_rest) in seq]
            assert kinds == sorted(kinds, reverse=True)                  # all head units, then all whole tiles
        # an even cut: no pair gets more than ceil(total / ranges) k-blocks of head work
        share = -(-sk_tiles * num_kb // ranges)
        for c in range(clusters):
            head = sum(kb1 - kb0 for (t, kb0, kb1, _s, _p) in units_of_cluster(c, clusters, full, sk_tiles, ranges, umax, num_kb) if t >= full)
            assert head <= share


def test_slab_exchange_is_order_independent_and_resets_its_ticket():
    # P parts publish f32 partials and take a ticket; whoever draws P - 1 adds the slabs in K order and zeroes the ticket
    rng = np.random.default_rng(3)
    order_matters = False
    for S in (2, 3, 4):
        partials = [rng.standard_normal(64).astype(np.float32) * (10.0 ** rng.integers(-3, 4)) for _ in range(S)]
        results = set()
        for order in itertools.permutations(range(S)):
            ticket, slabs, out = 0, {}, None
            for sl in order:                                     # arrival order of the parts
                slabs[sl] = partials[sl]                         # publish (threadfence) ...
                old, ticket = ticket, ticket + 1                 # ... then atomicAdd
                if old == S - 1:                                 # last arriver: ordered reduction, ticket left ready for the next launch
                    ticket = 0
                    acc = np.zeros(64, dtype=np.float32)
                    for i in range(S):
                        acc = (acc + slabs[i]).astype(np.float32)
                    out = acc
            assert ticket == 0 and out is not None
            results.add(out.tobytes())
        assert len(results) == 1                                 # bit-identical for every arrival order
        # an arrival-order sum would NOT be (f32 addition is not associative): that is what the ordered reduction buys
        naive = set()
        for order in itertools.permutations(range(S)):
            acc = np.zeros(64, dtype=np.float32)
            for i in order:
                acc = (acc + partials[i]).astype(np.float32)
            naive.add(acc.tobytes())
        order_matters |= len(naive) > 1
    assert order_matters


def test_host_policy_on_the_baseline_shapes():
    # (tiles, CTA pairs, k-blocks per tile) -> (tiles in the head, ranges)
    def head(tiles, clusters, num_kb):
        return host_plan(tiles, clusters, num_kb)[1:3]
    assert head(1024, 74, 128) == (0, 0)     # bf16 8192^3 on 256x256 tiles: 13.84 waves, nothing to gain
    assert head(256, 74, 128) == (34, 68)    # tf32 4096^3 (BASELINE config 2): 34 tiles in two equal halves each
    assert head(256, 74, 384) == (34, 68)    # 3xTF32 4096^3
    assert head(256, 74, 64) == (34, 68)     # bf16 4096^3 on 256x256 tiles
    # bf16 5120^3: 400 tiles of 256x256 = 5.41 waves -> modelled 5.75 with a head; the pair tile (3 whole waves of twice the work
    # at x1.06 = 5.66) still wins the variant choice, as measured (171.8 against 176.5 us)
    assert abs(host_plan(400, 74, 80)[0] - 5.75) < 1e-9 and 3 * 2 / 1.06 < 5.75
    assert head(8, 74, 256)[0] == 8          # 512^2 x 16384: the head is the whole problem, equal parts chosen by the model
    assert 2 <= head(8, 74, 256)[1] // 8 <= 8
    assert head(4, 74, 8) == (0, 0)          # tiny K: slices would be thinner than 8 k-blocks
    assert head(74, 74, 128) == (0, 0)       # exactly one wave
    t_with, *_ = host_plan(256, 74, 128)
    assert abs(t_with - (3 + 1.4 * 0.5 + 4.0 / 128)) < 1e-9
