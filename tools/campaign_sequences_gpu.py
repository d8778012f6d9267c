#!/usr/bin/env python3
"""Model-based sequence campaign on the GPU: long-lived renderers driven through random sequences of 20-40 calls -- the
setters, every one-call entry point (host and device), walked tickets held across later calls and rastered later on one
of two streams, world-1 sharded calls with and without a resolve, palette_lut_levels_device and Renderer.resolve on frames
rendered earlier, and deliberately refused calls -- against `Model`, a pure-Python restatement of DESIGN.md §3 ("Level
sets", "One host path per batch") and of the refusal rules.

The model tracks the renderer's own time and each level's sector moves, the compact state (compact_key) that each worklist
slot's own table set holds per timed level, the next ticket and the walked, unrastered tickets with the frames (pose, level,
tics, moves) they captured.  After every step the runner checks the launch count against the model, and that a refusal is
B2D_ERR_INVALID_ARG and launches nothing; after every rastered batch it checks the index and RGBA frames against the
oracle at the state the model says is in force, resolves against oracle/resolve.py, the poisoned guard bytes around every
device output, the status word and the table sets of the last walked batch (tables_at).  It also counts the *visible
stale events*: batches whose slot held another state that the oracle renders differently at the batch's poses, so that a
run which never exercises a stale table set cannot pass unnoticed.

    python tools/campaign_sequences_gpu.py [sequences] [--seed S] [--seq K] [-v]

`--seq K` re-runs sequence K of seed S alone; a mismatch prints the seed, the sequence, the step index and the steps."""
import argparse
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
if os.path.join(ROOT, "tools") not in sys.path:
    sys.path.insert(0, os.path.join(ROOT, "tools"))
import numpy as np  # noqa: E402

C2, RICH, SMALL, LARGE = range(4)          # tests/test_gpu_levels.py's four levels
STAGING_FRAMES = 1024                      # frame levels the first call of a level-staging user allocates for
TICS = (0, 9, 17, 35, 100, 1234, 77777, (1 << 31) + 5, (1 << 32) - 1)
RESOLVE_FORMATS = ("rgba", "rgb", "rgb_planar", "gray")

# one-call entry points: name -> (per-frame levels, per-frame states, timed, host frames)
CALLS = {
    "render": (False, False, False, True),
    "render_timed": (False, False, True, True),
    "render_states": (False, True, False, True),
    "render_levels": (True, False, False, True),
    "render_levels_states": (True, True, False, True),
    "render_device": (False, False, False, False),
    "render_device_timed": (False, False, True, False),
    "render_device_states": (False, True, False, False),
    "render_device_levels": (True, False, False, False),
    "render_device_levels_states": (True, True, False, False),
}
# walks (b2d_walk_device*): name -> (per-frame levels, per-frame states)
WALKS = {"walk_device": (False, False), "walk_device_states": (False, True), "walk_device_levels": (True, False),
         "walk_device_levels_states": (True, True)}
SHARDED = {"render_sharded": (False, False), "render_sharded_levels_states": (True, True)}
REFUSALS = ("pending_call", "pending_walk", "pending_sharded", "unknown_ticket", "rastered_ticket", "bad_level",
            "bad_range", "untimed_moves", "walk_too_big")


def step_kind(s):
    """the entry point a step calls (the setters by their ABI names)"""
    if s["op"] == "set_time":
        return "set_time_async" if s["async"] else "set_time"
    if s["op"] == "set_moves":
        return {"plain": "set_sector_moves", "async": "set_sector_moves_async", "level": "set_level_sector_moves"}[s["form"]]
    return s.get("entry", s["op"])


# ---- the model ---------------------------------------------------------------------------------------------------------
class Refused(Exception):
    """a call the library refuses with B2D_ERR_INVALID_ARG, before it launches or changes anything"""

    def __init__(self, kind):
        super().__init__(kind)
        self.kind = kind


class Model:
    """DESIGN.md §3 and the refusal rules, restated.  `timed[k]`: level k has time-dependent content or dynamic sectors
    (it has table sets); `dyn[k]`: it declares dynamic sectors; `key(k, tics, moves)`: the compact state of level k
    (equal keys, one table set).  Frames are (pose, level, tics, moves); moves a tuple of (sector, floor, ceil)."""

    def __init__(self, timed, dyn, key, max_batch):
        self.timed, self.dyn, self.key, self.mb = list(timed), list(dyn), key, int(max_batch)
        self.nlev = len(self.timed)
        self.T = 0
        self.M = [()] * self.nlev
        rest = {k: (key(k, 0, ()), 0, ()) for k in range(self.nlev) if self.timed[k]}
        self.slot = [dict(rest), dict(rest)]          # per worklist slot: level -> (key, tics, moves) its own set holds
        self.next_ticket = 0
        self.pending = {}                             # ticket -> walked batch, not rastered yet
        self.staging = {"lut": 0, "resolve": 0}       # frames each level staging holds
        self.events = set() if self.timed[0] else {"untimed_level0"}     # what the steps reached
        self._since = {}                              # pending ticket -> step kinds since its walk
        self._host_plain = False                      # a host call without RGBA has run
        self._host_rgba = False
        self._after_timed = False

    # -- the rules
    def _slot_busy(self, batches):
        """check_slots_free: the slots of the first min(batches, 2) tickets of a call hold no pending ticket"""
        for i in range(min(batches, 2)):
            if any((t & 1) == ((self.next_ticket + i) & 1) for t in self.pending):
                return True
        return False

    def _check_frames(self, levels, moves, bad_range):
        if levels is not None and any(int(k) >= self.nlev or int(k) < 0 for k in levels):
            raise Refused("bad_level")
        if bad_range:
            raise Refused("bad_range")
        if moves is not None:
            for i, mv in enumerate(moves):
                if mv and not self.dyn[int(levels[i]) if levels is not None else 0]:
                    raise Refused("untimed_moves")

    def _batch(self, frames, per_frame):
        """one walked batch into the next slot: -> its record (ticket, slot, frames, per_frame, launches, stale)"""
        slot = self.next_ticket & 1
        rec = dict(ticket=self.next_ticket, slot=slot, per_frame=per_frame, stale=[])
        self.next_ticket += 1
        if per_frame:
            rec["frames"] = list(frames)
            rec["launches"] = 2 + (1 if any(self.timed[f[1]] for f in frames) else 0)
            return rec
        used = sorted({f[1] for f in frames})
        for k in used:
            if self.timed[k]:
                key = self.key(k, self.T, self.M[k])
                held = self.slot[slot][k]
                if held[0] != key:
                    rec["stale"].append((k, held[1], held[2]))
                    self.slot[slot][k] = (key, self.T, self.M[k])
        rec["frames"] = [(p, k, self.T, self.M[k]) for p, k, _, _ in frames]
        rec["launches"] = 2 + len(rec["stale"])
        if rec["stale"]:
            if any(k >= 1 for k, _, _ in rec["stale"]):
                self.events.add("stale_level_ge1_slot%d" % slot)
        return rec

    def _frames(self, s, levels_arg, states_arg, timed_arg):
        n = len(s["poses"])
        lv = list(s["levels"]) if levels_arg else [0] * n
        if timed_arg:
            return [(s["poses"][i], 0, int(s["tics"][i]), self.M[0]) for i in range(n)]
        if states_arg:
            return [(s["poses"][i], int(lv[i]), int(s["tics"][i]), tuple(map(tuple, s["moves"][i]))) for i in range(n)]
        return [(s["poses"][i], int(lv[i]), None, None) for i in range(n)]

    def _batches(self, frames, size, per_frame):
        out = []
        for a in range(0, len(frames), size):
            out.append(self._batch(frames[a:a + size], per_frame))
            if a and out[-1]["stale"]:
                self.events.add("second_batch_stale")
        return out

    def _note_plain(self, per_frame):
        if self._after_timed and not per_frame:
            self.events.add("timed_then_plain")
        self._after_timed = False

    def step(self, s):
        """-> {launches, batches (walked and rastered now), walked (a held batch), rastered (a held batch), ticket}; raises
        Refused for a call the library refuses"""
        try:
            out = self._step(s)
        except Refused as e:
            self.events.add("refuse:" + e.kind)
            raise
        self.events.add("op:" + step_kind(s))
        if s["op"] in ("set_time", "set_moves"):
            for since in self._since.values():
                since.add("setter")
        return out

    def _step(self, s):
        op = s["op"]
        if op == "set_time":
            self.T = int(s["t"]) & 0xFFFFFFFF
            return dict(launches=0)
        if op == "set_moves":
            k = int(s["level"])
            if k < 0 or k >= self.nlev:
                raise Refused("bad_level")
            if s["moves"] and not self.dyn[k]:
                raise Refused("untimed_moves")
            self.M[k] = tuple(map(tuple, s["moves"]))
            return dict(launches=0)
        if op == "call":
            levels_arg, states_arg, timed_arg, host = CALLS[s["entry"]]
            n = len(s["poses"])
            self._check_frames(s["levels"] if levels_arg else None, s["moves"] if states_arg else None, s.get("bad_range"))
            if s["entry"] == "render_device" and n > self.mb:
                raise Refused("walk_too_big")
            nb = (n + self.mb - 1) // self.mb
            if self._slot_busy(nb):
                raise Refused("pending_call")
            per_frame = (states_arg or timed_arg) and (levels_arg or self.timed[0])
            frames = self._frames(s, levels_arg, states_arg, timed_arg)
            batches = self._batches(frames, self.mb, per_frame)
            self._note_plain(per_frame)
            if timed_arg:
                self.T = int(s["tics"][-1]) & 0xFFFFFFFF
                self._after_timed = True
            if host:
                if s.get("rgba") and not self._host_rgba and self._host_plain:
                    self.events.add("host_rgba_mid_sequence")
                self._host_rgba |= bool(s.get("rgba"))
                self._host_plain |= not s.get("rgba")
            return dict(launches=sum(b["launches"] for b in batches), batches=batches)
        if op == "walk":
            levels_arg, states_arg = WALKS[s["entry"]]
            n = len(s["poses"])
            if n == 0 or n > self.mb:
                raise Refused("walk_too_big")
            self._check_frames(s["levels"] if levels_arg else None, s["moves"] if states_arg else None, s.get("bad_range"))
            if self._slot_busy(1):
                raise Refused("pending_walk")
            per_frame = states_arg and (levels_arg or self.timed[0])
            rec = self._batch(self._frames(s, levels_arg, states_arg, False), per_frame)
            self._note_plain(per_frame)
            self._since[rec["ticket"]] = set()
            self.pending[rec["ticket"]] = rec
            return dict(launches=rec["launches"] - 1, walked=rec, ticket=rec["ticket"])
        if op == "raster":
            t = s["ticket"]
            if t not in self.pending:
                raise Refused("rastered_ticket" if t is not None and 0 <= t < self.next_ticket else "unknown_ticket")
            rec = self.pending.pop(t)
            if "setter" in self._since.pop(t):
                self.events.add("raster_after_setter")
            if any(u < t for u in self.pending):
                self.events.add("out_of_order")
            return dict(launches=1, rastered=rec)
        if op == "sharded":
            levels_arg, states_arg = SHARDED[s["entry"]]
            n = len(s["poses"])
            self._check_frames(s["levels"] if levels_arg else None, s["moves"] if states_arg else None, False)
            chunk = min(s["chunk"] or 256, self.mb, n)
            if self._slot_busy((n + chunk - 1) // chunk):
                raise Refused("pending_sharded")
            per_frame = states_arg                    # the level-set call always stages per-frame states
            batches = self._batches(self._frames(s, levels_arg, states_arg, False), chunk, per_frame)
            self._note_plain(per_frame)
            extra = len(batches) if s["resolve"] is not None else 0
            return dict(launches=sum(b["launches"] for b in batches) + extra, batches=batches)
        if op in ("lut", "resolve"):
            if s["levels"] is not None and any(int(k) >= self.nlev for k in s["levels"]):
                raise Refused("bad_level")
            n = int(s["n"])
            if s["levels"] is not None and n > self.staging[op]:
                cap = self.staging[op] or STAGING_FRAMES
                while cap < n:
                    cap *= 2
                if cap > STAGING_FRAMES:
                    self.events.add("staging_growth")
                self.staging[op] = cap
            return dict(launches=1)
        raise ValueError("unknown step %r" % op)


# ---- the levels ---------------------------------------------------------------------------------------------------------
def prepare_levels():
    """the four levels of tests/test_gpu_levels.py with what the campaign draws from: each level's oracle Level, its
    timed flag (campaign_levels_gpu.blob_info) and, on levels with dynamic sectors, a pool of move lists"""
    import campaign_levels_gpu as CL
    import rust_doom_b200 as b2d
    from oracle import wad as W
    from tests.test_gpu_levels import make_levels
    lvs = make_levels(b2d)
    for k, L in enumerate(lvs):
        L["level"] = W.Level(W.Archive(L["data"]), 0)
        L["doors"] = []
        L["timed"] = CL.blob_info(L["blob"])[1]
        pool = CL._moves_choices(L, np.random.default_rng(7 + k)) + [L["moves"]] if L["dyn"] else [[]]
        L["pool"] = [tuple(map(tuple, m)) for m in pool]
    return lvs


_KEYS = {}


def key_fn(lvs):
    """the compact_key of level k of `lvs` at (tics, moves), cached"""
    import campaign_levels_gpu as CL

    def key(k, tics, moves):
        kk = (id(lvs[k]["blob"]), int(tics) & 0xFFFFFFFF, tuple(moves))
        if kk not in _KEYS:
            _KEYS[kk] = CL.compact_key(lvs[k]["blob"], tics, moves)
        return _KEYS[kk]
    return key


def model_of(seq, lvs_all):
    lvs = [lvs_all[k] for k in seq["order"]]
    return Model([L["timed"] for L in lvs], [bool(L["dyn"]) for L in lvs], key_fn(lvs), seq["max_batch"])


# ---- the generator ------------------------------------------------------------------------------------------------------
def _view(rng):
    u = rng.random()
    if u < 0.45:
        return 160, 100
    if u < 0.8:
        return 320, 200
    if u < 0.9:
        return (32, 20) if rng.random() < 0.5 else (24, 16)
    return int(rng.integers(33, 200)), int(rng.integers(21, 120))


def _factors(w, h):
    return [f for f in range(1, 9) if w % f == 0 and h % f == 0]


class _Gen:
    def __init__(self, rng, seq, lvs_all):
        self.rng, self.seq = rng, seq
        self.lvs = [lvs_all[k] for k in seq["order"]]
        self.nlev = len(self.lvs)
        self.model = model_of(seq, lvs_all)
        self.walks = {}                                # tag -> ticket of walks the model accepted
        self.frames_made = False

    def pick(self, xs):
        return xs[int(self.rng.integers(0, len(xs)))]

    def tic(self):
        u = self.rng.random()
        if u < 0.25:                                   # a state a slot may already hold
            return int(self.pick([0, self.model.T] + [v[1] for s in self.model.slot for v in s.values()]))
        return int(self.pick(TICS)) if u < 0.8 else int(self.rng.integers(0, 1 << 32))

    def frames(self, n, levels_arg, states_arg):
        rng = self.rng
        lv = [int(rng.integers(0, self.nlev)) if levels_arg else 0 for _ in range(n)]
        poses = [int(self.pick(self.seq["pool"][k])) for k in lv]
        tics = [self.tic() for _ in range(n)]
        moves = [list(self.pick(self.lvs[k]["pool"])) if states_arg else [] for k in lv]
        return dict(poses=poses, levels=lv, tics=tics, moves=moves)

    def n(self, cap=3):
        return int(self.rng.integers(1, cap * self.seq["max_batch"] + 1))

    def setter(self):
        rng = self.rng
        u = rng.random()
        if u < 0.45:
            return dict(op="set_time", t=self.tic(), **{"async": bool(rng.random() < 0.3)})
        dynl = [k for k in range(self.nlev) if self.lvs[k]["dyn"]]
        k = self.pick(dynl) if dynl and rng.random() < 0.85 else int(rng.integers(0, self.nlev))
        mv = list(self.pick(self.lvs[k]["pool"]))
        form = "level" if k else self.pick(["plain", "async", "level"])
        return dict(op="set_moves", level=k, moves=mv, form=form)

    def call(self, entry=None, n=None):
        entry = entry or self.pick(list(CALLS))
        levels_arg, states_arg, timed_arg, host = CALLS[entry]
        n = n or (int(self.rng.integers(1, self.seq["max_batch"] + 1)) if entry == "render_device" else self.n())
        s = dict(op="call", entry=entry, rgba=bool(self.rng.random() < 0.35), **self.frames(n, levels_arg, states_arg))
        return s

    def walk(self, entry=None):
        entry = entry or self.pick(list(WALKS))
        levels_arg, states_arg = WALKS[entry]
        n = int(self.rng.integers(1, self.seq["max_batch"] + 1))
        return dict(op="walk", entry=entry, tag=len(self.seq["steps"]), **self.frames(n, levels_arg, states_arg))

    def raster(self):
        pend = sorted(t for t in self.model.pending)
        if not pend:
            return None
        t = pend[-1] if len(pend) > 1 and self.rng.random() < 0.5 else pend[0]
        tag = [g for g, tt in self.walks.items() if tt == t][0]
        return dict(op="raster", tag=tag, ticket=t, stream=int(self.rng.integers(0, 2)), rgba=bool(self.rng.random() < 0.3))

    def sharded(self):
        rng = self.rng
        entry = self.pick(list(SHARDED))
        levels_arg, states_arg = SHARDED[entry]
        n = self.n()
        res = None
        if rng.random() < 0.5:
            res = (int(self.pick(_factors(self.seq["w"], self.seq["h"]))), self.pick(RESOLVE_FORMATS))
        return dict(op="sharded", entry=entry, chunk=int(rng.integers(0, self.seq["max_batch"] + 3)), resolve=res,
                    **self.frames(n, levels_arg, states_arg))

    def staging(self):
        if not self.frames_made:
            return None
        rng = self.rng
        big = self.seq["w"] * self.seq["h"] <= 640 and rng.random() < 0.5
        n = int(rng.integers(STAGING_FRAMES + 1, 2 * STAGING_FRAMES + 100)) if big else int(rng.integers(1, 12))
        levels = [int(k) for k in rng.integers(0, self.nlev, n)]
        if rng.random() < 0.5:
            return dict(op="lut", n=n, levels=levels, offset=4 * int(rng.integers(0, 4)))
        return dict(op="resolve", n=n, levels=levels if rng.random() < 0.7 else None,
                    factor=int(self.pick(_factors(self.seq["w"], self.seq["h"]))), fmt=self.pick(RESOLVE_FORMATS))

    def refusal(self):
        """a call the library must refuse, of a kind drawn from those that apply now"""
        m, rng = self.model, self.rng
        kinds = ["unknown_ticket", "bad_level", "bad_range", "walk_too_big"]
        if m.pending:
            kinds += ["pending_call", "pending_sharded"]
        if any((t & 1) == (m.next_ticket & 1) for t in m.pending):
            kinds.append("pending_walk")
        if m.next_ticket > len(m.pending):
            kinds.append("rastered_ticket")
        if not self.lvs[0]["dyn"]:
            kinds.append("untimed_moves")
        kind = self.pick(kinds)
        if kind == "pending_call":
            busy = [(t & 1) for t in m.pending]
            n = self.seq["max_batch"] * (1 if (m.next_ticket & 1) in busy else 2)
            return self.call(self.pick(["render", "render_levels_states", "render_device_levels", "render_device_timed",
                                        "render_timed", "render_device_states"]), n)
        if kind == "pending_sharded":
            s = self.sharded()
            n = 2 * self.seq["max_batch"]
            s.update(chunk=0, **self.frames(n, *SHARDED[s["entry"]]))
            return s
        if kind == "pending_walk":
            return self.walk()
        if kind == "unknown_ticket":
            return dict(op="raster", tag=None, ticket=self.pick([-1, m.next_ticket, m.next_ticket + 7]), stream=0, rgba=False)
        if kind == "rastered_ticket":
            done = [t for t in range(m.next_ticket) if t not in m.pending]
            return dict(op="raster", tag=None, ticket=self.pick(done[-3:]), stream=1, rgba=False)
        if kind == "bad_level":
            u = rng.random()
            if u < 0.5:
                s = self.call(self.pick([e for e, v in CALLS.items() if v[0]])) if u < 0.3 else self.walk(
                    self.pick(["walk_device_levels", "walk_device_levels_states"]))
                s["levels"][int(rng.integers(0, len(s["levels"])))] = self.nlev
                return s
            if u < 0.7 and self.frames_made:
                s = self.staging()
                if s and s["levels"] is not None:
                    s["levels"][int(rng.integers(0, s["n"]))] = self.nlev
                    return s
            return dict(op="set_moves", level=self.nlev if rng.random() < 0.7 else -1, moves=[], form="level")
        if kind == "bad_range":
            s = self.call("render_states", int(rng.integers(1, self.seq["max_batch"] + 1)))
            s["bad_range"] = True
            return s
        if kind == "untimed_moves":
            return dict(op="set_moves", level=0, moves=[(0, 8, 0)], form=self.pick(["plain", "async"]))
        s = self.walk()                                 # walk_too_big
        s.update(**self.frames(self.seq["max_batch"] + 1, *WALKS[s["entry"]]))
        return s

    def add(self, s):
        """append the step and advance the model"""
        if s is None:
            return
        self.seq["steps"].append(s)
        try:
            out = self.model.step(s)
        except Refused:
            return
        if s["op"] == "walk":
            self.walks[s["tag"]] = out["ticket"]
        if s["op"] in ("call", "raster") or (s["op"] == "sharded" and s["resolve"] is None):
            self.frames_made = True            # the runner keeps them for the palette and resolve steps


def draw_sequence(seed, k, lvs_all):
    """sequence k of a campaign seeded `seed`: {order (indices into the four levels), single, max_batch, w, h, fov, pool
    (pose indices per renderer level), poses (the pose table, POSE_DTYPE), steps}"""
    import rust_doom_b200 as b2d
    from tests.conftest import sample_poses
    rng = np.random.default_rng([seed, k])
    first = int(rng.choice([C2, RICH, SMALL]))
    single = bool(rng.random() < 0.3)
    if single:
        order = [first]
    else:
        rest = [j for j in range(4) if j != first]
        rng.shuffle(rest)
        order = [first] + [int(j) for j in rest[:int(rng.integers(1, 4))]]
    w, h = _view(rng)
    seq = dict(seed=seed, k=k, order=order, single=single, max_batch=int(rng.integers(1, 6)), w=w, h=h, fov=65.0, steps=[])
    poses, pool = [], []
    for j, lk in enumerate(order):
        p = sample_poses(b2d, lvs_all[lk]["scene"], 6, 1000 * k + 17 * lk + seed % 1000)
        pool.append(list(range(len(poses), len(poses) + len(p))))
        poses.extend(p)
    seq["poses"], seq["pool"] = np.array(poses, dtype=b2d.POSE_DTYPE), pool
    g = _Gen(rng, seq, lvs_all)
    n_steps = int(rng.integers(20, 41))
    while len(seq["steps"]) < n_steps:
        u = rng.random()
        if u < 0.2:
            g.add(g.setter())
        elif u < 0.47:
            g.add(g.call())
        elif u < 0.62:
            g.add(g.walk())
        elif u < 0.77:
            g.add(g.raster())
        elif u < 0.83:
            g.add(g.sharded())
        elif u < 0.91:
            g.add(g.staging())
        else:
            g.add(g.refusal())
    for t in sorted(g.model.pending):                 # leave no ticket behind
        g.add(dict(op="raster", tag=[a for a, b in g.walks.items() if b == t][0], ticket=t, stream=t & 1, rgba=False))
    return seq


class Forced(_Gen):
    """a sequence written step by step: frames given as (renderer level, pose of that level's pool)"""

    def __init__(self, lvs_all, order, max_batch, w=160, h=100, single=False, seed=7):
        import rust_doom_b200 as b2d
        from tests.conftest import sample_poses
        seq = dict(seed=seed, k=0, order=list(order), single=single, max_batch=max_batch, w=w, h=h, fov=65.0, steps=[])
        poses, pool = [], []
        for lk in order:
            p = sample_poses(b2d, lvs_all[lk]["scene"], 6, seed + 17 * lk)
            pool.append(list(range(len(poses), len(poses) + len(p))))
            poses.extend(p)
        seq["poses"], seq["pool"] = np.array(poses, dtype=b2d.POSE_DTYPE), pool
        super().__init__(np.random.default_rng(seed), seq, lvs_all)

    def _fr(self, frames, tics=None, moves=None):
        n = len(frames)
        return dict(poses=[self.seq["pool"][k][j % len(self.seq["pool"][k])] for k, j in frames], levels=[k for k, _ in frames],
                    tics=list(tics) if tics is not None else [0] * n, moves=[list(m) for m in moves] if moves else [[]] * n)

    def set_time(self, t):
        self.add(dict(op="set_time", t=t, **{"async": False}))
        return self

    def set_moves(self, level, moves, form="level"):
        self.add(dict(op="set_moves", level=level, moves=list(moves), form=form))
        return self

    def do(self, entry, frames, tics=None, moves=None, rgba=False, **kw):
        s = dict(op="call", entry=entry, rgba=rgba, **self._fr(frames, tics, moves))
        if entry in WALKS:
            s = dict(op="walk", entry=entry, tag=len(self.seq["steps"]), **self._fr(frames, tics, moves))
        elif entry in SHARDED:
            s = dict(op="sharded", entry=entry, chunk=kw.get("chunk", 0), resolve=kw.get("resolve"), **self._fr(frames, tics, moves))
        self.add(s)
        return s.get("tag")

    def raster(self, tag, stream=0, rgba=False):
        self.add(dict(op="raster", tag=tag, ticket=self.walks[tag], stream=stream, rgba=rgba))
        return self

    def staging(self, op, n, levels=None, factor=1, fmt="rgba"):
        s = dict(op=op, n=n, levels=levels, offset=4) if op == "lut" else \
            dict(op=op, n=n, levels=levels, factor=factor, fmt=fmt)
        self.add(s)
        return self


FORCED = ("stale_sets_in_both_slots", "held_ticket_across_a_timed_call", "untimed_level0_render_timed",
          "per_frame_between_plain_batches", "sharded_between_device_calls", "level_staging_growth")


def forced_sequences(lvs_all):
    """[(name, sequence)] in FORCED order: one written-out sequence per history the random draw may reach rarely"""
    out = []
    # 1. the two slots hold different stale sets of RICH (level 1); a three-batch host call crosses both
    f = Forced(lvs_all, [C2, RICH, SMALL], 2)
    f.set_time(1234).do("render_levels", [(1, 0)])
    f.set_time(77777).do("render_levels", [(1, 1)])
    f.set_moves(1, lvs_all[RICH]["moves"]).set_time(9)
    f.do("render_levels", [(1, 2), (0, 0), (1, 3), (1, 4), (2, 0), (1, 5)], rgba=True)
    f.do("render_levels", [(1, 0), (1, 1), (0, 1)])
    out.append(("stale_sets_in_both_slots", f.seq))
    # 2. a ticket walked into slot 0 and held: two-batch calls (slots 1 and 0) are refused, a one-batch timed call goes to
    #    slot 1, then a one-batch call (slot 0) is refused; the held ticket, rastered after setters and the timed call,
    #    shows its walk's state
    f = Forced(lvs_all, [RICH], 2, single=True)
    f.set_time(1234).set_moves(0, lvs_all[RICH]["moves"], "plain")
    held = f.do("walk_device", [(0, 0), (0, 1)])
    f.set_moves(0, [], "async").set_time(77777)
    f.do("render", [(0, 0), (0, 1), (0, 2)])
    f.do("render_sharded", [(0, 0), (0, 1), (0, 2)])
    f.do("render_device_timed", [(0, 2)], tics=[35])
    f.do("render_device", [(0, 3)])
    f.raster(held, stream=1)
    f.do("render", [(0, 0), (0, 1), (0, 2)], rgba=True)
    out.append(("held_ticket_across_a_timed_call", f.seq))
    # 3. an untimed level 0: render_timed is plain (two launches per batch) and still moves the time RICH's next batch reads
    f = Forced(lvs_all, [SMALL, RICH, C2], 2)
    f.do("render_levels", [(1, 0), (2, 0)])
    f.do("render_timed", [(0, 0), (0, 1), (0, 2)], tics=[5, 9, 1234])
    f.do("render_levels", [(1, 1), (1, 2)])
    f.do("render_device_levels", [(2, 1), (1, 3)])
    out.append(("untimed_level0_render_timed", f.seq))
    # 4. a per-frame batch between plain batches on a level set: its slot's own sets are neither read nor changed
    f = Forced(lvs_all, [C2, RICH, LARGE], 3)
    f.set_time(100).do("render_device_levels", [(0, 0), (1, 0), (2, 0)])
    f.do("render_device_levels_states", [(1, 1), (2, 1), (0, 1)], tics=[77777, 9, 1234], moves=[lvs_all[RICH]["moves"], [], []])
    f.do("render_device_levels", [(1, 2), (2, 2), (0, 2)])
    f.do("render_levels", [(2, 3), (0, 3), (1, 3)])
    f.do("walk_device_levels_states", [(1, 4), (1, 5)], tics=[100, 101], moves=[[], lvs_all[RICH]["moves"]])
    f.raster(f.seq["steps"][-1]["tag"])
    f.do("render_levels", [(1, 4), (0, 4)])
    out.append(("per_frame_between_plain_batches", f.seq))
    # 5. world-1 sharded calls between device calls: the ticket parity after them, resolved and not, refused while a
    #    ticket is pending
    f = Forced(lvs_all, [C2, RICH], 2)
    f.do("render_device", [(0, 0)])
    f.set_time(1234).do("render_sharded", [(0, 0), (0, 1), (0, 2)])
    held = f.do("walk_device", [(0, 3)])
    f.do("render_sharded", [(0, 0), (0, 1), (0, 2), (0, 3)], resolve=(2, "rgb_planar"))
    f.do("render_sharded_levels_states", [(0, 0), (1, 1)], tics=[3, 4], chunk=1)
    f.raster(held)
    f.set_time(77777).do("render_sharded_levels_states", [(1, 0), (0, 1), (1, 2)], tics=[9, 9, 1234], chunk=1, resolve=(4, "gray"))
    f.do("render_sharded", [(0, 4), (0, 5)], resolve=(1, "rgba"))
    f.do("render_device_levels", [(1, 4), (0, 4), (0, 5)])
    held = f.do("walk_device_levels", [(1, 5)])
    f.raster(held, stream=1)
    out.append(("sharded_between_device_calls", f.seq))
    # 6. the level staging of palette_lut_levels_device and resolve_device grows past 1024 frames, and serves smaller calls
    f = Forced(lvs_all, [C2, RICH, SMALL], 4, w=32, h=20)
    f.do("render_levels", [(0, 0), (1, 0), (2, 0), (1, 1), (2, 1)])
    lv = [k % 3 for k in range(2000)]
    f.staging("lut", 10, lv[:10]).staging("lut", 1500, lv[:1500]).staging("lut", 7, lv[1:8])
    f.staging("resolve", 20, lv[:20], 2, "rgb").staging("resolve", 2000, lv, 4, "gray").staging("resolve", 3, lv[2:5], 1, "rgba")
    f.staging("resolve", 5, None, 2, "rgb_planar")
    f.do("render_device_levels", [(1, 2), (2, 2)])
    f.staging("lut", 1100, lv[:1100])
    out.append(("level_staging_growth", f.seq))
    return out


def describe_step(i, s):
    d = {k: v for k, v in s.items() if k not in ("op", "poses", "levels", "tics", "moves")}
    if "poses" in s:
        d["n"] = len(s["poses"])
        d["levels"] = s["levels"][:8] if s.get("levels") is not None else None
        if s["op"] != "walk" or WALKS[s["entry"]][1]:
            d["tics"] = s["tics"][:4]
    elif s["op"] in ("lut", "resolve") and s["levels"] is not None:
        d["levels"] = s["levels"][:6]
    if s["op"] == "set_moves":
        d["moves"] = s["moves"][:3]
    return "%3d %s %s" % (i, s.get("entry", s["op"]), d)


def describe(seq):
    return "%s renderer of levels %s, %dx%d, max_batch %d, %d steps" % (
        "single-level" if seq["single"] else "level-set", seq["order"], seq["w"], seq["h"], seq["max_batch"], len(seq["steps"]))


# ---- the runner ---------------------------------------------------------------------------------------------------------
def run_sequence(seq, lvs_all, stats=None):
    """-> list of problems (the first failing step's); stats (dict) accumulates steps, frames, visible stale events"""
    import torch
    import campaign_levels_gpu as CL
    import rust_doom_b200 as b2d
    from oracle import resolve as RES, scene as S
    from rust_doom_b200 import _lib
    from tests.test_gpu_levels import _palette
    from tests.test_gpu_levels_states import check_level_sets
    from tests.test_gpu_states import check_state_sets
    stats = {} if stats is None else stats
    for key in ("steps", "frames", "refused", "stale", "visible_stale"):
        stats.setdefault(key, 0)
    lvs = [lvs_all[k] for k in seq["order"]]
    timed = [L["timed"] for L in lvs]
    w, h, mb = seq["w"], seq["h"], seq["max_batch"]
    npix = w * h
    view = b2d.make_view(w, h, seq["fov"])
    r = b2d.Renderer(lvs[0]["scene"], view, max_batch=mb) if seq["single"] else \
        b2d.Renderer.from_levels([L["scene"] for L in lvs], view, max_batch=mb)
    model = model_of(seq, lvs_all)
    orc = CL._Oracle(lvs, w, h, seq["fov"])
    pals = [_palette(L["scene"]) for L in lvs]
    playpals = [L["scene"].palette_rgb() for L in lvs]
    gen = torch.Generator(device="cuda")
    gen.manual_seed(seq["seed"] * 1000 + seq["k"])
    s_walk, s_r, s_dev = torch.cuda.Stream(priority=-1), (torch.cuda.Stream(), torch.cuda.Stream()), torch.cuda.Stream()
    keep, tickets = [], {}                       # device poses of held walks; tag -> ticket the library returned
    bank = None                                  # (index frames, levels) of the last rendered frames
    L = _lib.load()

    def dev_poses(s):
        p = np.ascontiguousarray(seq["poses"][s["poses"]])
        t = torch.from_numpy(p.view(np.int32).reshape(-1, 4).copy()).cuda()
        keep.append(t)
        return t.data_ptr()

    def oracle_of(frames, rgba):
        p = seq["poses"][[f[0] for f in frames]]
        return orc.frames(p, [f[1] for f in frames], [f[2] for f in frames], [list(f[3]) for f in frames], rgba)

    def check_batches(batches, idx, col, what):
        """frames of walked-and-rastered batches against the oracle at the model's state; visible stale events"""
        frames = [f for b in batches for f in b["frames"]]
        want, want_rgba = oracle_of(frames, col is not None)
        bad = [(i, int((want[i] != idx[i]).sum())) for i in range(len(frames)) if not np.array_equal(want[i], idx[i])]
        out = ["%s: index frames differ from the oracle at the model's state (frame, pixels): %s" % (what, bad[:6])] if bad else []
        if col is not None:
            badc = [i for i in range(len(frames)) if not np.array_equal(want_rgba[i], col[i].view(np.uint32))]
            if badc:
                out.append("%s: RGBA frames differ: %s" % (what, badc[:6]))
        a = 0
        for b in batches:
            if b["stale"]:
                stats["stale"] += 1
                old = {k: (t, mv) for k, t, mv in b["stale"]}
                sel = [i for i, f in enumerate(b["frames"]) if f[1] in old]
                prev = [(f[0], f[1], old[f[1]][0], old[f[1]][1]) for f in (b["frames"][i] for i in sel)]
                then, _ = oracle_of(prev, False)
                if any(not np.array_equal(then[j], want[a + i]) for j, i in enumerate(sel)):
                    stats["visible_stale"] += 1
            a += len(b["frames"])
        stats["frames"] += len(frames)
        return out, want

    def check_sets(batches, step_levels_arg):
        """the table sets of the last walked batch against tables_at"""
        b = batches[-1]
        fr = b["frames"]
        if b["per_frame"]:
            lv = [f[1] for f in fr]
            if step_levels_arg:
                check_level_sets(r, lvs, timed, lv, [f[2] for f in fr], [list(f[3]) for f in fr], len(fr))
            elif timed[0]:
                check_state_sets(r, lvs[0]["blob"], [f[2] for f in fr], [list(f[3]) for f in fr], len(fr))
        elif timed[0] and any(f[1] == 0 for f in fr):
            f = [f for f in fr if f[1] == 0][0]
            if r.state_tables(0) != S.tables_at(lvs[0]["blob"], f[2], list(f[3])):
                return ["the level-0 table set of the last plain batch is not tables_at(%d, %s)" % (f[2], list(f[3])[:3])]
        return []

    def guarded_out(n, rgba):
        gi = CL._Guarded(n * npix, max(n, mb) * npix, 0, gen)
        gc = CL._Guarded(n * npix * 4, max(n, mb) * npix * 4, 0, gen) if rgba else None
        return gi, gc

    def guards_ok(gs):
        out = []
        for what, g in gs:
            t = g.touched() if g is not None else []
            if t:
                out.append("%s: guard bytes written at offsets %s" % (what, t))
        return out

    problems = []
    for i, s in enumerate(seq["steps"]):
        stats["steps"] += 1
        try:
            pred = model.step(s)
            refused = None
        except Refused as e:
            pred, refused = dict(launches=0), e.kind
        l0 = r.launch_count
        err = None
        res = {}
        try:
            res = _execute(r, s, seq, L, dev_poses, guarded_out, tickets, bank, (s_walk, s_r, s_dev), gen)
        except b2d.B2dError as e:
            err = e
        except BaseException as e:                         # noqa: BLE001 -- report, do not crash the campaign
            if isinstance(e, KeyboardInterrupt):
                raise
            err = e
        dl = r.launch_count - l0
        if refused is not None:
            stats["refused"] += 1
            if not isinstance(err, b2d.B2dError) or err.code != b2d.ERR_INVALID_ARG:
                problems.append("step %d: the model refuses it (%s), the library returned %s" % (i, refused, err or "OK"))
        elif err is not None:
            problems.append("step %d: %s: %s" % (i, type(err).__name__, str(err).splitlines()[0] if str(err) else ""))
        if dl != pred["launches"]:
            problems.append("step %d: %d launches, the model gives %d" % (i, dl, pred["launches"]))
        if problems:
            break
        if refused is not None:
            continue
        try:
            if "ticket" in pred and res.get("ticket") != pred["ticket"]:
                problems.append("step %d: ticket %s, the model gives %d" % (i, res.get("ticket"), pred["ticket"]))
            if s["op"] == "walk":
                tickets[s["tag"]] = res["ticket"]
            batches = pred.get("batches") or ([pred["rastered"]] if "rastered" in pred else [])
            if s["op"] in ("call", "walk", "sharded"):
                problems += check_sets(pred.get("batches") or [pred["walked"]], (CALLS.get(s["entry"]) or WALKS.get(s["entry"])
                                                                                or SHARDED[s["entry"]])[0])
            if batches and "index" in res:
                torch.cuda.synchronize()
                idx, col = res["index"](), res["rgba"]() if res.get("rgba") else None
                if res.get("resolve"):
                    factor, fmt = res["resolve"]
                    frames = [f for b in batches for f in b["frames"]]
                    want, _ = oracle_of(frames, False)
                    lv = [f[1] for f in frames] if s["entry"] == "render_sharded_levels_states" else None
                    ref = RES.resolve(want, playpals, factor, fmt, lv)
                    if np.ascontiguousarray(ref).tobytes() != idx.tobytes():
                        problems.append("step %d: resolved sharded frames differ from oracle/resolve.py" % i)
                    stats["frames"] += len(frames)
                else:
                    p, want = check_batches(batches, idx, col, "step %d" % i)
                    problems += p
                    bank = (want, np.array([f[1] for b in batches for f in b["frames"]], np.uint32))
                problems += guards_ok(res.get("guards", []))
                st = r.status()
                if st:
                    problems.append("step %d: status %d" % (i, st))
            if s["op"] in ("lut", "resolve") and refused is None:
                torch.cuda.synchronize()
                src = res["src"]
                lv = np.zeros(len(src), np.int64) if s["levels"] is None else np.asarray(s["levels"])
                if s["op"] == "lut":
                    want = np.stack([pals[int(lv[f])][src[f]] for f in range(len(src))])
                    got = res["index"]().view(np.uint32)
                else:
                    want = RES.resolve(src, playpals, s["factor"], s["fmt"], s["levels"])
                    got = res["index"]()
                    if s["fmt"] == "rgba":
                        got = got.view(np.uint32)
                if not np.array_equal(want, got):
                    problems.append("step %d: %s output differs from the oracle" % (i, s["op"]))
                problems += guards_ok(res.get("guards", []))
        except BaseException as e:                         # noqa: BLE001 -- check_level_sets' failure, a library error
            if isinstance(e, KeyboardInterrupt):
                raise
            problems.append("step %d: %s: %s" % (i, type(e).__name__, str(e).splitlines()[0] if str(e) else ""))
        if problems:
            break
    torch.cuda.synchronize()
    r.close()
    if problems:
        problems = [p for p in problems] + ["steps:"] + [describe_step(j, st) for j, st in enumerate(seq["steps"][:i + 1])]
    return problems


def _execute(r, s, seq, L, dev_poses, guarded_out, tickets, bank, streams, gen):
    """enqueue one step as an application would -> {ticket, index (callable -> host frames), rgba, guards, src, resolve}"""
    import torch
    import campaign_levels_gpu as CL
    import rust_doom_b200 as b2d
    from rust_doom_b200 import _frame_states
    s_walk, s_r, s_dev = streams
    op, w, h, mb = s["op"], seq["w"], seq["h"], seq["max_batch"]
    npix = w * h

    def after_inputs():
        """the library's streams see the poses and outputs made on torch's stream (an event each, no host wait)"""
        for st in (s_walk, s_dev) + tuple(s_r):
            st.wait_stream(torch.cuda.current_stream())
    if op == "set_time":
        if s["async"]:
            r.set_time_async(s["t"], s_walk.cuda_stream)
        else:
            r.set_time(s["t"])
        return {}
    if op == "set_moves":
        if s["form"] == "level":
            r.set_level_sector_moves(s["level"], s["moves"])
        else:
            r.set_sector_moves(s["moves"], stream=s_walk.cuda_stream if s["form"] == "async" else None)
        return {}
    if op == "call":
        entry, n, rgba = s["entry"], len(s["poses"]), s["rgba"]
        levels_arg, states_arg, timed_arg, host = CALLS[entry]
        lv, tics, moves = s["levels"], np.array(s["tics"], np.uint64).astype(np.uint32), s["moves"]
        if host:
            poses = np.ascontiguousarray(seq["poses"][s["poses"]])
            if s.get("bad_range"):                     # a frame's move range runs past the end of the move list
                states, arr, nm = _frame_states(tics, None, n)
                states[n - 1].first_move, states[n - 1].n_moves = 0, 1
                out = np.empty((n, h, w), np.uint8)
                rc = L.b2d_render_states(r._h, poses.ctypes.data, states, n, arr, 0, out.ctypes.data, None)
                if rc < 0:
                    raise b2d.B2dError(rc, "")
                return {}
            got = {"render": lambda: r.render(poses, rgba=rgba),
                   "render_timed": lambda: r.render_timed(poses, tics, rgba=rgba),
                   "render_states": lambda: r.render_states(poses, tics, moves, rgba=rgba),
                   "render_levels": lambda: r.render_levels(poses, lv, rgba=rgba),
                   "render_levels_states": lambda: r.render_levels_states(poses, lv, tics, moves, rgba=rgba)}[entry]()
            idx, col = got if rgba else (got, None)
            return dict(index=lambda: idx, rgba=(lambda: col) if rgba else None)
        dp = dev_poses(s)
        gi, gc = guarded_out(n, rgba)
        o, oc, st = gi.ptr, gc.ptr if gc else 0, s_dev.cuda_stream
        after_inputs()
        {"render_device": lambda: r.render_device(dp, n, o, oc, st),
         "render_device_timed": lambda: r.render_device_timed(dp, tics, n, o, oc, st),
         "render_device_states": lambda: r.render_device_states(dp, tics, n, o, oc, moves, st),
         "render_device_levels": lambda: r.render_device_levels(dp, lv, n, o, oc, st),
         "render_device_levels_states": lambda: r.render_device_levels_states(dp, lv, tics, n, o, oc, moves, st)}[entry]()
        return dict(index=lambda: gi.frames(n, h, w, torch.uint8), rgba=(lambda: gc.frames(n, h, w, torch.int32)) if gc else None,
                    guards=[("index", gi), ("rgba", gc)])
    if op == "walk":
        entry, n = s["entry"], len(s["poses"])
        lv, tics, moves = s["levels"], np.array(s["tics"], np.uint64).astype(np.uint32), s["moves"]
        dp, st = dev_poses(s), s_walk.cuda_stream
        after_inputs()
        t = {"walk_device": lambda: r.walk_device(dp, n, st),
             "walk_device_states": lambda: r.walk_device_states(dp, tics, n, moves, st),
             "walk_device_levels": lambda: r.walk_device_levels(dp, lv, n, st),
             "walk_device_levels_states": lambda: r.walk_device_levels_states(dp, lv, tics, n, moves, st)}[entry]()
        return dict(ticket=t)
    if op == "raster":
        ticket = tickets.get(s["tag"], s["ticket"]) if s["tag"] is not None else s["ticket"]
        walk = [x for x in seq["steps"] if x["op"] == "walk" and x["tag"] == s["tag"]]
        n = len(walk[0]["poses"]) if walk else mb
        gi, gc = guarded_out(n, s["rgba"])
        after_inputs()
        r.raster_device(ticket, gi.ptr, gc.ptr if gc else 0, s_r[s["stream"]].cuda_stream)
        return dict(index=lambda: gi.frames(n, h, w, torch.uint8), rgba=(lambda: gc.frames(n, h, w, torch.int32)) if gc else None,
                    guards=[("index", gi), ("rgba", gc)])
    if op == "sharded":
        n, poses = len(s["poses"]), np.ascontiguousarray(seq["poses"][s["poses"]])
        res = s["resolve"]
        fb = r.resolve_frame_bytes(res[0], b2d.RESOLVE_FORMATS[res[1]]) if res else npix
        out = np.zeros(n * fb, np.uint8)

        class _Dev:
            def __init__(self, ptr, nb):
                self.__cuda_array_interface__ = {"shape": (nb,), "typestr": "|u1", "data": (ptr, False), "version": 2}

        def on_chunk(k, first, cnt, ptr, ranks, stream):
            with torch.cuda.stream(torch.cuda.ExternalStream(stream)):
                out[first * fb:(first + cnt) * fb] = torch.as_tensor(_Dev(ptr, cnt * fb), device="cuda").cpu().numpy()
        if s["entry"] == "render_sharded":
            r.render_sharded(CL._comm(), poses, s["chunk"], on_chunk=on_chunk, resolve=res)
        else:
            r.render_sharded_levels_states(CL._comm(), poses, s["levels"], np.array(s["tics"], np.uint64).astype(np.uint32),
                                           s["moves"], s["chunk"], on_chunk=on_chunk, resolve=res)
        return dict(index=lambda: out if res else out.reshape(n, h, w), resolve=res)
    if op in ("lut", "resolve"):
        n = s["n"]
        src_frames, _ = bank
        src = np.resize(src_frames, (n, h, w))
        dsrc = torch.from_numpy(src).cuda()
        if op == "lut":
            gl = CL._Guarded(n * npix * 4, n * npix * 4, s["offset"], gen)
            after_inputs()
            r.palette_lut_levels_device(dsrc.data_ptr(), s["levels"], n, gl.ptr, s_dev.cuda_stream)
            return dict(src=src, index=lambda: gl.frames(n, h, w, torch.int32), guards=[("palette_lut_levels_device", gl)])
        out = r.resolve(dsrc, s["factor"], s["fmt"], s["levels"])
        return dict(src=src, index=lambda: out.cpu().numpy())
    raise ValueError(op)


def run(seqs, seed=12345, only=None, verbose=False, todo=None, lvs=None):
    """-> (sequences run, mismatching, stats, seconds); `todo`: [(label, sequence)] instead of the seeded draw"""
    t0 = time.time()
    lvs = prepare_levels() if lvs is None else lvs
    if todo is None:
        todo = [(only, draw_sequence(seed, only, lvs))] if only is not None else \
            [(k, draw_sequence(seed, k, lvs)) for k in range(seqs)]
    bad, stats = 0, {}
    for k, seq in todo:
        problems = run_sequence(seq, lvs, stats)
        if problems:
            bad += 1
            print("MISMATCH --seed %d --seq %s: %s" % (seed, k, describe(seq)), flush=True)
            for p in problems:
                print("    " + p, flush=True)
        elif verbose:
            print("ok  sequence %s: %s" % (k, describe(seq)), flush=True)
    return len(todo), bad, stats, time.time() - t0


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("sequences", nargs="?", type=int, default=100)
    ap.add_argument("--seed", type=int, default=12345)
    ap.add_argument("--seq", type=int, default=None)
    ap.add_argument("-v", action="store_true")
    a = ap.parse_args()
    n, bad, st, secs = run(a.sequences, a.seed, a.seq, a.v)
    print("sequence campaign: %d sequences, %d mismatching, %d steps (%d refused), %d frames, %d stale-set batches "
          "(%d visible), %.1f s" % (n, bad, st.get("steps", 0), st.get("refused", 0), st.get("frames", 0), st.get("stale", 0),
                                    st.get("visible_stale", 0), secs))
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
