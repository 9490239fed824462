"""The work items of a pruned window sweep (csrc/karto_sweep_plan.cuh: split_chunks<4, 32>, split_range<4>,
chunk_groups): a match that lists few angles splits each angle's groups I0..I3 E0..E3 into beam ranges cut on multiples
of 4, which k_sweep_window<LISTED> sums in shared memory.  Checked on the host, without a GPU (tests/sweep_plan_check.cu):
every listed beam lies in exactly one range, every range boundary and every part of a group starts on a multiple of 4,
empty groups included, and the split keeps about two items per warp within the accumulators that fit."""
import numpy as np

from test_sweep_plan import CFG2, CFG2_SEARCH, plan, plan_request  # noqa: F401 (plan: the driver fixture)

WARPS = 16  # WIN_THREADS / 32


def check_split(C, counts, items):
    """the C items of an angle whose groups hold `counts` beams cover each listed beam once, on multiples of 4"""
    assert len(items) == C
    starts = np.concatenate([[0], np.cumsum(counts)])
    seen = np.zeros(int(starts[-1]), dtype=np.int64)
    prev_hi = 0
    for it in items:
        lo, hi, parts = it[0], it[1], it[2:]
        assert lo == prev_hi and lo <= hi and lo % 4 == 0 and hi % 4 == 0, it
        prev_hi = hi
        covered = 0
        for g in range(8):
            off, ln = parts[2 * g], parts[2 * g + 1]
            assert off % 4 == 0 and ln % 4 == 0 and ln >= 0, (g, it)
            assert ln == 0 or 0 <= off and off + ln <= counts[g], (g, it, counts)
            if ln:
                assert lo <= starts[g] + off and starts[g] + off + ln <= hi, (g, it)
            seen[starts[g] + off:starts[g] + off + ln] += 1
            covered += ln
        assert covered == hi - lo, it
    assert prev_hi == starts[-1]
    assert (seen == 1).all()


def group_counts(rng, n):
    """8 group lengths, multiples of 4, summing to at most n rounded up to 4, with empty groups among them"""
    w = rng.random(8) * (rng.random(8) < 0.7)
    q = (n + 3) // 4
    c = np.floor(w / max(w.sum(), 1e-12) * q).astype(int) * 4
    return [int(v) for v in c]


def test_every_listed_beam_in_exactly_one_range(plan):
    rng = np.random.default_rng(5)
    cases = []
    for n in (1, 3, 4, 5, 31, 33, 64, 1081, 4500, 9000):
        for listed in (1, 2, 3, 15, 16, 17, 31, 32, 181, 1024):
            C = plan([f"chunks 4 {listed} {n} {WARPS} 16"])[0]["chunks"]
            for counts in ([0] * 8, [4 * ((n + 3) // 4)] + [0] * 7, [0] * 7 + [4 * ((n + 3) // 4)], group_counts(rng, n),
                           group_counts(rng, n)):
                cases.append((C, counts))
    for C in (2, 3, 7, 16, 32, 33):  # more ranges than quads of beams: empty ranges
        cases.append((C, [4, 0, 0, 8, 0, 0, 4, 0]))
    out = plan([f"split {C} " + " ".join(map(str, counts)) for C, counts in cases])
    for (C, counts), r in zip(cases, out):
        check_split(C, counts, r["items"])


def test_chunk_rule(plan):
    reqs, want = [], []
    for n in range(1, 9001, 97):
        for listed in list(range(1, 40)) + [181, 1024]:
            for slots in (0, 1, 15, 16, 31):
                reqs.append(f"chunks 4 {listed} {n} {WARPS} {slots}")
                want.append((listed, n, slots))
    for (listed, n, slots), r in zip(want, plan(reqs)):
        C = r["chunks"]
        assert C >= 1
        if listed > slots or n < 64:  # the planes do not fit, or too few beams for two ranges: one item per angle
            assert C == 1, (listed, n, slots, C)
            continue
        assert listed * C >= 2 * WARPS or C == n // 32, (listed, n, slots, C)  # about two items per warp
        assert listed * (C - 1) < 2 * WARPS, (listed, n, slots, C)           # and no more ranges than that needs
        assert n // C >= 32, (listed, n, slots, C)                            # at least 32 beams per range on average


def test_cfg2_lists_fit_the_accumulators(plan):
    """at the benchmark's shape (a 165 KB grid, 31 x 31 candidates) the 16 probe angles are split in two"""
    (pl,) = plan([plan_request(CFG2, 1081, 1024, CFG2_SEARCH)])
    assert pl["prune"] and pl["acc_slots"] == 16, pl
    assert pl["listed_smem"] == pl["win_smem"] + 16 * 31 * 31 * 4 and pl["listed_smem"] + 3200 + 512 <= 232448, pl
    out = plan([f"chunks 4 {listed} 1081 {WARPS} {pl['acc_slots']}" for listed in (16, 2, 1, 3, 17)])
    assert [r["chunks"] for r in out] == [2, 16, 32, 11, 1]
