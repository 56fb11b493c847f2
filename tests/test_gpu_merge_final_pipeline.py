"""k_merge_final's tile pipeline: a tile's look-back and emit run one iteration after its resolve, and the CTA's last tile is
finished after the loop.  These cases stress what that creates -- many tiles per CTA with look-backs deeper than one warp's
window (one CTA per SM), a CTA whose only tile is finished after the loop, and jobs of exactly one and two tiles -- against
the oracle."""
import os

import numpy as np
import pytest

from dbeel_b200 import capi, sstable
from dbeel_b200 import workloads as W

from helpers import BASE_TS, assert_run_equal, model_compact
from test_gpu_merge_final import test_groups_straddling_merge_tiles as _straddling
from test_gpu_parity import check_against_oracle

pytestmark = pytest.mark.gpu

FIN_NOMINAL = 1792 - 64  # records per tile of the last merge level (kFinNominal)


def _engine(env):
    old = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        return capi.Engine(0)
    finally:
        for k, v in old.items():
            if v is None:
                del os.environ[k]
            else:
                os.environ[k] = v


@pytest.fixture(scope="module")
def engine_one_cta():
    """One k_merge_final CTA per SM: the scaled benchmark shapes give every CTA several tiles, and the nearest predecessor
    holding an inclusive prefix is often more than 128 tiles back."""
    eng = _engine({"DBEEL_FUSED_FINAL": "1", "DBEEL_FIN_CTAS_RT": "1"})
    yield eng
    eng.close()


@pytest.fixture(scope="module")
def engine_default_ctas():
    eng = _engine({"DBEEL_FUSED_FINAL": "1"})
    yield eng
    eng.close()


@pytest.mark.parametrize("cfg,keys", [(W.CFG2, 250_000), (W.CFG3, 50_000)])
def test_many_tiles_per_cta(engine_one_cta, cfg, keys):
    c = W.scaled(cfg, keys)
    check_against_oracle(engine_one_cta, W.make_merge_runs(c), c.keep_tombstones, what=c.name + " one CTA per SM")
    check_against_oracle(engine_one_cta, W.make_merge_runs(c, equal_ts=True), c.keep_tombstones,
                         what=c.name + " equal ts, one CTA per SM")


@pytest.mark.parametrize("seed", range(2))
def test_straddling_groups_one_cta(engine_one_cta, seed):
    _straddling(engine_one_cta, seed)


def _two_runs(rng, total):
    """Two runs of `total` entries between them that share about a third of their keys (groups of two across the merge),
    with tombstones and equal timestamps among the duplicates."""
    n0 = total // 2
    n1 = total - n0
    shared = max(0, min(n0, n1) // 3)
    pool = [b"p%07d" % i for i in range(0, 4 * total + 8, 2)]
    picks = rng.permutation(len(pool))
    k0 = [pool[i] for i in picks[:n0]]
    k1 = k0[:shared] + [pool[i] for i in picks[n0:n0 + n1 - shared]]
    runs = []
    for keys in (k0, k1):
        ents = []
        for k in sorted(keys):
            v = b"" if rng.random() < 0.15 else bytes(rng.integers(0, 256, int(rng.integers(1, 60)), dtype=np.uint8))
            ents.append((k, v, BASE_TS + int(rng.integers(0, 3))))
        runs.append(sstable.build_run(ents))
    return runs


@pytest.mark.parametrize("total", [2, 1000, FIN_NOMINAL, FIN_NOMINAL + 1, 3000, 2 * FIN_NOMINAL])
@pytest.mark.parametrize("which", ["default", "one_cta"])
def test_one_and_two_tiles(engine_default_ctas, engine_one_cta, which, total):
    """Up to FIN_NOMINAL records the last level is one tile, which only the drain after the loop finishes; up to twice that
    it is two, each finished by the drain of the CTA that holds it."""
    eng = engine_default_ctas if which == "default" else engine_one_cta
    rng = np.random.default_rng(total)
    runs = _two_runs(rng, total)
    for keep in (False, True):
        gd, gi, _, n = check_against_oracle(eng, runs, keep, what=f"{total} entries keep={keep}")
        exp, en = model_compact(runs, keep)
        assert n == en
        assert_run_equal((gd, gi), exp, f"{total} entries vs model")
        assert eng.stats()["merge_passes"] == 1
