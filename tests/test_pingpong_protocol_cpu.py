"""CPU: the ping-pong pipeline protocol of the tile engine (tile_gemm.cuh, gemm_consumer_pingpong), modelled in
tests/pingpong_model.py, over every CTA schedule the plan builds and over designed edge cases; and the model's own
sensitivity: every deliberately broken protocol fails."""
import pytest

from tests import pingpong_model as pm

SEEDS = range(4)


def _check(n_tiles, nkb, stages, seeds=SEEDS):
    for seed in seeds:
        r = pm.run_protocol(n_tiles, nkb, stages, seed=seed)
        assert r["ok"], (n_tiles, nkb, stages, seed, r["error"])
        assert r["turns"] == [i % 2 for i in range(n_tiles)]


def test_plan_schedules_run_to_completion():
    """Every (tiles per CTA, k-blocks per tile, ring depth) of every ping-pong launch at batches 1, 2, 5, 64, 129 and 512,
    in every operand mode, with and without the parity top-down launches."""
    cases = pm.pingpong_schedules()
    assert len(cases) > 20
    assert any(n == 1 for n, _, _ in cases) and any(n % 2 == 1 and n > 1 for n, _, _ in cases)
    assert any(n % 2 == 0 for n, _, _ in cases)
    assert {s for _, _, s in cases} == {2, 4}             # three and two pieces (one-piece modes never ping-pong)
    for n, nkb, stages in sorted(cases):
        _check(n, nkb, stages, seeds=[n * 1009 + nkb])


def test_plan_selection():
    """Which launches are ping-pong: fragment epilogues outside halo mode with more than one product and at most 32
    k-blocks per tile; the fp32 heads, halo layers, long-K layers and one-piece modes are not."""
    for mode, P in pm.MODES.items():
        for B in (2, 5, 64, 129, 512):
            geo = {ln.layer + (f"@{ln.parity}" if ln.parity else "") + ("@sparse" if ln.sparse else ""): pm.geometry(ln, P)
                   for ln in pm.network(B)}
            for name, g in geo.items():
                if name.startswith(("heat", "mlp2")) or P == 1 or g["k_blocks"] > 32:
                    assert not g["pingpong"], name
                if g["pingpong"]:
                    assert g["block_n"] == 64 and g["stages"] >= 2 and not g["halo"], name
            if P == 1:
                continue
            assert not geo["lat6"]["pingpong"] and not geo["s4u1c2"]["pingpong"]     # 144 and 72 k-blocks
            assert geo["stem"]["pingpong"] and geo["s1u1c3"]["pingpong"] and geo["s2u1c1"]["pingpong"]
            assert geo["b0_p3td_u"]["pingpong"] and geo["b0_p3td"]["pingpong"] and geo["fusion"]["pingpong"]
            if P == 2:
                assert not geo["s2u1c2"]["pingpong"]             # halo mode
                assert geo["s1u2c3"]["stages"] == 4              # 48 KiB slots in two-piece modes


@pytest.mark.parametrize("n_tiles,nkb,stages", [
    (1, 1, 2), (1, 4, 4), (1, 9, 2),        # one tile in the CTA (warpgroup 1 never gets a turn)
    (2, 1, 2), (2, 2, 4), (4, 3, 3),        # even counts
    (3, 1, 2), (3, 2, 4), (5, 5, 3), (7, 2, 2),   # odd counts
    (6, 1, 8), (9, 1, 2), (8, 144, 4),
])
def test_designed_cases(n_tiles, nkb, stages):
    _check(n_tiles, nkb, stages)


@pytest.mark.parametrize("total,grid", [(1, 1), (132, 132), (10, 7), (200, 132), (265, 132), (9, 5)])
def test_designed_grids(total, grid):
    """1 tile in total, 1 tile per CTA, and grids larger than half the tiles: every CTA's sequence from the enumeration."""
    counts = [pm.cta_tiles(total, b, grid) for b in range(grid)]
    assert sum(counts) == total and min(counts) >= 1
    seen = sorted(pm.tile_index(total, b, grid, i) for b in range(grid) for i in range(counts[b]))
    assert seen == list(range(total))                          # every tile belongs to exactly one CTA
    for n in set(counts):
        _check(n, 2, 3)


def _errors(faults, cases):
    """Every error the broken protocol meets over the cases and 40 schedules each ("" when none)."""
    errs = set()
    for n, nkb, stages in cases:
        for seed in range(40):
            r = pm.run_protocol(n, nkb, stages, seed=seed, faults=faults)
            if not r["ok"]:
                errs.add(r["error"])
    return " | ".join(sorted(errs))


def test_broken_protocols_fail():
    cases = [(1, 1, 2), (2, 1, 2), (3, 2, 4), (6, 1, 4), (5, 3, 3), (9, 1, 2)]
    err = _errors(pm.Faults(early_handover=True), cases)
    assert "not read in the producer's order" in err, err
    for f in (pm.Faults(skip_last_release=True), pm.Faults(empty_count=2), pm.Faults(turn_without_tile=True)):
        err = _errors(f, cases)
        assert "deadlock" in err, (f, err)
    assert _errors(pm.Faults(), cases) == ""
