"""No GPU: the model of tools/campaign_sequences_gpu.py against the rules DESIGN.md §3 states and the hand-written GPU tests
pin -- the launch lists of tests/test_gpu_renderer_state.py, tests/test_gpu_states_scale.py and tests/test_gpu_levels.py and
the refusals of tests/test_gpu_stream_order.py -- and what the sequences of tests/test_gpu_campaign_sequences.py reach:
every step kind, every refusal kind and the histories that decide which table set a batch reads."""
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if os.path.join(ROOT, "tools") not in sys.path:
    sys.path.insert(0, os.path.join(ROOT, "tools"))
import campaign_sequences_gpu as Q  # noqa: E402

SHUT = ((3, 0, -72),)                  # a move list (the model only compares keys)


def _simple(timed=(True,), dyn=(True,), max_batch=4):
    """a model whose compact state is the whole (tics, moves)"""
    return Q.Model(timed, dyn, lambda k, t, m: (int(t) & 0xFFFFFFFF, tuple(m)), max_batch)


def _frames(n, levels=None, tics=None, moves=None):
    return dict(poses=list(range(n)), levels=list(levels) if levels is not None else [0] * n,
                tics=list(tics) if tics is not None else [0] * n, moves=[list(m) for m in moves] if moves else [[]] * n)


def call(entry, n, **kw):
    return dict(op="call", entry=entry, rgba=False, **_frames(n, **kw))


def walk(entry, n, tag=0, **kw):
    return dict(op="walk", entry=entry, tag=tag, **_frames(n, **kw))


def sharded(entry, n, chunk, **kw):
    return dict(op="sharded", entry=entry, chunk=chunk, resolve=None, **_frames(n, **kw))


def launches(m, *steps):
    return [m.step(s)["launches"] for s in steps]


def test_model_setters_and_each_slot_expanding_once():
    """test_setters_enqueue_nothing_and_each_slot_expands_once: [2, 2], the setters 0, [3, 3, 2, 2], 3, [2, 3]"""
    m = _simple(max_batch=4)
    b = call("render_device", 4)
    assert launches(m, b, b) == [2, 2]
    assert launches(m, dict(op="set_time", t=1000, **{"async": False}), dict(op="set_moves", level=0, moves=SHUT, form="plain"),
                    dict(op="set_time", t=1000, **{"async": True}), dict(op="set_moves", level=0, moves=SHUT, form="async")) == [0] * 4
    assert launches(m, b, b, b, b) == [3, 3, 2, 2]
    m.step(dict(op="set_time", t=2000, **{"async": False}))
    assert launches(m, b) == [3]
    m.step(dict(op="set_time", t=1000, **{"async": False}))
    assert launches(m, b, b) == [2, 3]


def test_model_slots_shared_by_plain_and_per_frame_batches():
    """test_slots_shared_by_plain_and_per_frame_batches: [2, 2, 1, 1, 2, 1, 2, 1, 1, 1], and the plain ticket walked at A
    keeps A's frames while the renderer is at B"""
    m = _simple(max_batch=8)
    m.step(dict(op="set_time", t=300, **{"async": False}))
    m.step(dict(op="set_moves", level=0, moves=SHUT, form="plain"))
    got = [m.step(walk("walk_device", 8))]
    m.step(dict(op="set_time", t=(1 << 32) - 3, **{"async": False}))
    m.step(dict(op="set_moves", level=0, moves=(), form="plain"))
    got.append(m.step(walk("walk_device_states", 8, tics=range(7, 47, 5))))
    got.append(m.step(dict(op="raster", ticket=1)))
    got.append(m.step(dict(op="raster", ticket=0)))
    assert got[-1]["rastered"]["frames"][0][2:] == (300, SHUT)
    for t in (2, 3, 4):
        got.append(m.step(walk("walk_device", 8)))
        got.append(m.step(dict(op="raster", ticket=t)))
    assert [g["launches"] for g in got] == [2, 2, 1, 1, 2, 1, 2, 1, 1, 1]
    assert "out_of_order" in m.events


@pytest.fixture(scope="module")
def lvs(b2d):
    return Q.prepare_levels()


def test_model_levels_launch_counts(lvs):
    """test_levels_launch_counts on the four levels, with the real compact states: two launches per batch at a fixed
    state, then one per stale timed level the batch uses in its slot"""
    C2, RICH, SMALL, LARGE = range(4)
    timed = [L["timed"] for L in lvs]
    assert timed[C2] and timed[RICH] and not timed[SMALL]
    m = Q.Model(timed, [bool(L["dyn"]) for L in lvs], Q.key_fn(lvs), 16)

    def batch(lv):
        return m.step(call("render_device_levels", len(lv), levels=lv))["launches"]

    mix = [0, 1, 2, 3] * 4
    assert [batch(mix) for _ in range(4)] == [2, 2, 2, 2]
    m.step(dict(op="set_time", t=500, **{"async": False}))
    got = [batch([0, 2] * 8), batch(mix), batch([1, 3] * 8), batch(mix), batch(mix)]
    assert got == [3, 2 + sum(timed), 2 + timed[1] + timed[3], 2, 2]
    m.step(dict(op="set_moves", level=RICH, moves=lvs[RICH]["moves"], form="level"))
    assert [batch([0, 2] * 8), batch([1] * 16), batch(mix), batch(mix)] == [2, 3, 3, 2]


def test_model_refuses_one_call_renders_over_a_pending_ticket():
    """test_one_call_renders_refuse_a_pending_ticket: with a ticket walked into slot 0 and held, every two-batch one-call
    render and the two-chunk sharded calls are refused with no launch and no change; one batch into the free slot is
    accepted; then one batch is refused too (the next slot is the pending ticket's); the ticket then rasters"""
    m = _simple(timed=(True, True, False), dyn=(True, False, False), max_batch=8)
    t = m.step(walk("walk_device_levels_states", 6, levels=[0, 1, 2, 0, 1, 2]))["ticket"]
    lv = [0, 1, 2] * 4
    before = (m.next_ticket, dict(m.pending), [dict(s) for s in m.slot], m.T)
    for s in (call("render", 12), call("render_timed", 12, tics=range(12)), call("render_states", 12),
              call("render_levels", 12, levels=lv), call("render_levels_states", 12, levels=lv),
              call("render_device_timed", 12, tics=range(12)), call("render_device_states", 12),
              call("render_device_levels", 12, levels=lv), call("render_device_levels_states", 12, levels=lv),
              sharded("render_sharded", 12, 6), sharded("render_sharded_levels_states", 12, 6, levels=lv)):
        with pytest.raises(Q.Refused):
            m.step(s)
    assert (m.next_ticket, dict(m.pending), [dict(s) for s in m.slot], m.T) == before
    assert m.step(call("render_levels_states", 6, levels=[0, 1, 2, 2, 1, 0]))["launches"] == 3
    with pytest.raises(Q.Refused) as e:
        m.step(call("render_device", 6))
    assert e.value.kind == "pending_call"
    assert m.step(dict(op="raster", ticket=t))["launches"] == 1
    with pytest.raises(Q.Refused) as e:
        m.step(dict(op="raster", ticket=t))
    assert e.value.kind == "rastered_ticket"


def test_model_timed_calls():
    """a *_timed call renders frame i at tics[i] with the current level-0 moves and leaves the renderer at tics[n-1]; on
    an untimed level 0 its batches are plain, and the time still moves for the other levels"""
    m = _simple(timed=(True,), max_batch=2)
    m.step(dict(op="set_moves", level=0, moves=SHUT, form="plain"))
    out = m.step(call("render_timed", 3, tics=[5, 9, 1234]))
    assert [f[2:] for b in out["batches"] for f in b["frames"]] == [(5, SHUT), (9, SHUT), (1234, SHUT)]
    assert out["launches"] == 6 and m.T == 1234
    m = _simple(timed=(False, True), dyn=(False, True), max_batch=2)
    assert m.step(call("render_device_timed", 3, tics=[5, 9, 1234]))["launches"] == 4 and m.T == 1234
    out = m.step(call("render_levels", 2, levels=[1, 1]))
    assert out["launches"] == 2 + 1 and out["batches"][0]["frames"][0][2] == 1234
    assert "timed_then_plain" in m.events and "untimed_level0" in m.events


def test_model_argument_refusals():
    m = _simple(timed=(False, True), dyn=(False, True), max_batch=3)
    cases = [(call("render_levels", 2, levels=[0, 2]), "bad_level"), (walk("walk_device", 4), "walk_too_big"),
             (dict(op="set_moves", level=0, moves=SHUT, form="plain"), "untimed_moves"),
             (dict(op="set_moves", level=2, moves=(), form="level"), "bad_level"),
             (dict(call("render_states", 2), bad_range=True), "bad_range"),
             (dict(op="raster", ticket=0), "unknown_ticket"), (dict(op="lut", n=4, levels=[0, 1, 2, 0]), "bad_level")]
    for s, kind in cases:
        with pytest.raises(Q.Refused) as e:
            m.step(s)
        assert e.value.kind == kind
    assert m.next_ticket == 0 and m.T == 0


@pytest.fixture(scope="module")
def reached(lvs):
    """the events the model records over the GPU test's short run and its forced sequences"""
    from tests.test_gpu_campaign_sequences import short_run
    events = set()
    for _, seq in short_run(lvs) + Q.forced_sequences(lvs):
        m = Q.model_of(seq, lvs)
        for s in seq["steps"]:
            try:
                m.step(s)
            except Q.Refused:
                pass
        assert not m.pending, "a sequence leaves a ticket unrastered"
        events |= m.events
    return events


def test_short_run_reaches_every_step_and_refusal_kind(reached):
    steps = list(Q.CALLS) + list(Q.WALKS) + list(Q.SHARDED) + ["raster", "lut", "resolve", "set_time", "set_time_async",
                                                                "set_sector_moves", "set_sector_moves_async",
                                                                "set_level_sector_moves"]
    assert not [s for s in steps if "op:" + s not in reached]
    assert not [k for k in Q.REFUSALS if "refuse:" + k not in reached]


def test_short_run_reaches_the_histories(reached):
    """a stale set of a level >= 1 in each slot, a held ticket rastered after a setter, tickets rastered out of order, a
    multi-batch call whose second batch lands in a stale slot, a timed call followed by a plain call, an untimed level 0,
    host RGBA first requested mid-sequence and level-staging growth"""
    want = ["stale_level_ge1_slot0", "stale_level_ge1_slot1", "raster_after_setter", "out_of_order", "second_batch_stale",
            "timed_then_plain", "untimed_level0", "host_rgba_mid_sequence", "staging_growth"]
    assert not [w for w in want if w not in reached]


def test_forced_sequences(lvs):
    """each written-out sequence does what its name says in the model"""
    seqs = dict(Q.forced_sequences(lvs))
    assert tuple(seqs) == Q.FORCED

    def trace(name):
        seq = seqs[name]
        m = Q.model_of(seq, lvs)
        out = []
        for s in seq["steps"]:
            try:
                out.append(m.step(s))
            except Q.Refused as e:
                out.append(e.kind)
        return out

    t = trace("stale_sets_in_both_slots")
    stale = [b["stale"] for b in t[6]["batches"]]
    assert [(k, tics) for k, tics, _ in stale[0]] == [(0, 0), (1, 1234)] and stale[2] == []
    assert [(k, tics) for k, tics, _ in stale[1]] == [(1, 77777)]
    t = trace("held_ticket_across_a_timed_call")
    assert t[5:7] == ["pending_call", "pending_sharded"] and t[7]["batches"][0]["slot"] == 1 and t[8] == "pending_call"
    assert t[9]["rastered"]["frames"][0][2:] == (1234, tuple(map(tuple, lvs[Q.RICH]["moves"])))
    t = trace("untimed_level0_render_timed")
    assert [x["launches"] for x in t] == [2, 4, 3, 4]
    t = trace("sharded_between_device_calls")
    assert t[3]["ticket"] == 3 and t[4:6] == ["pending_sharded", "pending_sharded"]
    assert t[-2]["ticket"] == 10
    t = trace("level_staging_growth")
    assert all(isinstance(x, dict) for x in t)
