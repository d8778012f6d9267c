"""-m gpu: the sequence campaign of tools/campaign_sequences_gpu.py.  Long-lived renderers driven through random sequences
of setters, one-call renders, held walks, sharded calls at world 1, palette and resolve calls and refused calls, each step
checked against the campaign's model of the renderer's time, sector moves, worklist slots and tickets: launches, refusals,
frames against the oracle at the state the model says is in force, table sets, guard bytes and the status word.  Then one
written-out sequence per history that decides what a batch reads.  tests/test_campaign_sequences.py checks, without a GPU,
that the model restates the hand-written launch counts and that these sequences reach every step and refusal kind."""
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if os.path.join(ROOT, "tools") not in sys.path:
    sys.path.insert(0, os.path.join(ROOT, "tools"))
import campaign_sequences_gpu as Q  # noqa: E402

pytestmark = pytest.mark.gpu

SEED, SEQUENCES = 2026, 60
MIN_VISIBLE_STALE = 45          # batches of the short run whose slot held a state the oracle renders differently


def short_run(lvs):
    """[(label, sequence)] of the deterministic random run"""
    return [(k, Q.draw_sequence(SEED, k, lvs)) for k in range(SEQUENCES)]


@pytest.fixture(scope="module")
def lvs(b2d):
    return Q.prepare_levels()


def test_campaign_sequences_short_run(b2d, lvs):
    """60 random sequences of SEED: no mismatching step, and enough stale table sets that show in the frames"""
    n, bad, stats, secs = Q.run(0, SEED, todo=short_run(lvs), lvs=lvs)
    print("%d sequences, %d mismatching, %s, %.1f s" % (n, bad, stats, secs))
    assert bad == 0, "%d of %d sequences differ (printed above)" % (bad, n)
    assert stats["visible_stale"] >= MIN_VISIBLE_STALE, stats


@pytest.mark.parametrize("name", Q.FORCED)
def test_campaign_sequences_forced(b2d, lvs, name):
    """one written-out sequence: its every step as the model says"""
    seq = dict(Q.forced_sequences(lvs))[name]
    problems = Q.run_sequence(seq, lvs)
    assert not problems, "\n".join(problems)
