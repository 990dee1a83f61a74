"""Quorum and vote counting of every step kernel against the rule restated in a few lines, one crafted group per case.

ra_server.erl counts members three ways: the commit index a leader may move to (evaluate_quorum /
increment_commit_index :3606-3630 over agreed_commit(match_indexes) :3644-3661), whether a candidate or a pre-voter
has its quorum (handle_candidate :1026-1044, handle_pre_vote :1212-1229 against required_quorum / count_voters
:3969-3982) and what a consistent query's heartbeat round agreed on (agreed_commit(query_indexes) :3632-3642).  The
kernels count with a sorting network as wide as the specialisation (3, 5 or 7 registers, 8 in the runtime-M and the
general kernel, zero-padded), an exact shortcut for "nothing moves", a 32-bit pass and voter masks, so a group's size
picks the code.  For every M from 1 to 8 the table holds

- commit cases: a leader in every slot, every voter mask of the other slots (sampled where 2^(M-1) is large), match
  indexes and last_written drawn around commit_index (one below, equal, one and two above, often all tied), the
  current term's run starting below, at or above the rank-nth candidate (the §5.4.2 gate open or closed); the event
  is a successful AppendEntries reply from a voter, a non-voter or a slot outside the group, or a WRITTEN;
- vote cases: candidates and pre-voters with 0..M-1 votes, every voter mask, the member itself a voter or not; the
  event is one granted vote or pre-vote;
- query cases: a leader's own and its peers' query indexes; the event is one heartbeat reply.

One step, then what each backend reads back must equal the rule, and the emulation's and the engine's rows, records,
notes, counters and query state must equal the oracle's.  Settings: routed with the 32-bit and the 64-bit hot kernel
(M = 3, 5, 7 run their own specialisations, other M the runtime-M kernel), host-routed (the TR_HOST kernel at M = 5),
pure (every event in the general kernel) and the same table moved past 2^30 and 2^32, where the 32-bit pass refuses
the rows and the 64-bit kernels take them.
"""
import random

import pytest

from emu_lib import Emu
from fuzz_lib import TABLE_SETTINGS as SETTINGS, compare, observe, shift_event, shift_state
from oracle_lib import Oracle
from ra_b200 import abi
from ra_suite import clone, make_backend

T, C0 = 7, 10                                   # current term and commit_index of the crafted rows
VALS = [C0 - 1, C0, C0 + 1, C0 + 2]             # match indexes, last_written, reply indexes
LAST = C0 + 2                                   # a leader's last index

# SETTINGS, name: (engine config, RA_STEP_WIDE, (index shift, term shift) or None, leaders' replies stay in the hot kernel)
MEMBERS = list(range(1, abi.RA_MAX_MEMBERS + 1))


# ---- the rule, restated ---------------------------------------------------------------------------------------------
def agreed_commit(indexes):
    """agreed_commit/1: sorted descending, element trunc(N/2)+1 (1-based)"""
    return sorted(indexes, reverse=True)[len(indexes) // 2]


def required_quorum(n_voters):
    """required_quorum/1: trunc(count_voters/2)+1"""
    return n_voters // 2 + 1


def term_at(s, i):
    """fetch_term/2 on the row's log view (no snapshot here): the term of the run holding i, None outside the log"""
    if s.n_runs == 0 or not s.first_index <= i <= s.last_index:
        return None
    return [s.run_term[k] for k in range(s.n_runs) if s.run_start[k] <= i][-1]


def expected_commit(s, base):
    """increment_commit_index/1 on the read-back row s: agreed_commit over [last_written | voter peers' match
    indexes] when the entry there is of the current term, else the commit index the case was loaded with"""
    idx = [s.last_written_index] + [s.peers[p].match_index for p in range(s.n_members)
                                    if p != s.self_slot and s.peers[p].voter]
    cand = agreed_commit(idx)
    return cand if term_at(s, cand) == s.current_term else base


# ---- the cases ------------------------------------------------------------------------------------------------------
class Case:
    def __init__(self, kind, state, event, desc, query=None):
        self.kind, self.state, self.event, self.desc, self.query = kind, state, event, desc, query
        self.votes, self.member_voter = state.votes, state.membership == abi.VOTER


def _mask_desc(s):
    return "".join("V" if s.peers[p].voter else "-" for p in range(s.n_members))


def _member(m, me):
    s = abi.empty_row(0, 1, m)                  # (table() assigns the row)
    s.self_slot = me
    return s


def _leader(m, me, voters, rng, cur_run):
    """A leader at slot `me` whose log is 1..LAST: term T-3 up to 3, T-1 after, T from cur_run on (none if past
    LAST); voters: the other slots that vote."""
    s = _member(m, me)
    abi.set_log(s, [(i, T if i >= cur_run else (T - 3 if i < 4 else T - 1)) for i in range(1, LAST + 1)])
    s.role, s.current_term, s.leader_slot, s.voted_for = abi.LEADER, T, me, me
    s.commit_index, s.last_applied = C0, C0 - 2
    tied = rng.random() < 0.2
    v0 = rng.choice(VALS)
    s.last_written_index = v0 if tied else rng.choice(VALS)
    s.last_written_term = term_at(s, s.last_written_index)
    for p in range(m):
        pe = s.peers[p]
        pe.commit_index_sent = C0
        if p == me:
            pe.voter, pe.next_index, pe.match_index = 1, LAST + 1, 0
        else:
            pe.voter = 1 if p in voters else 0
            pe.match_index = v0 if tied else rng.choice(VALS)
            pe.next_index = pe.match_index + 1
    return s


def _masks(n_slots, rng, cap=64):
    """every subset of n_slots slots as a bit mask, or `cap` of them drawn (with the empty and the full one)"""
    full = (1 << n_slots) - 1
    if full + 1 <= cap:
        return list(range(full + 1))
    return [0, full] + rng.sample(range(1, full), cap - 2)


def commit_cases(m, rng):
    """(state, event) of leaders: every leader slot and voter mask of the others, with a reply from a voter, a
    non-voter, a slot outside the group, or a WRITTEN"""
    out = []
    for me in range(m):
        others = [p for p in range(m) if p != me]
        masks = _masks(len(others), rng, 64 if m < 8 else 24)
        for mask in masks * max(1, 48 // (m * len(masks))):      # (small groups: several draws per mask)
            voters = {p for k, p in enumerate(others) if mask >> k & 1}
            kinds = ["written", "unknown"] + (["voter", "voter"] if voters else []) + \
                (["nonvoter"] if len(voters) < len(others) else [])
            for kind in kinds:
                s = _leader(m, me, voters, rng, rng.choice([C0 - 1, C0, C0 + 1, C0 + 2, C0 + 3]))
                b = rng.choice(VALS)
                if kind == "written":
                    ev = abi.ev_written(0, term_at(s, b), b, b)
                else:
                    f = (rng.choice(sorted(voters)) if kind == "voter" else
                         rng.choice([p for p in others if p not in voters]) if kind == "nonvoter" else
                         rng.choice([m, 9, 14]))
                    ev = abi.ev_aer_reply(0, f, T, True, b + 1, b, term_at(s, b))
                desc = ("leader slot %d voters %s last_written %d match %s, current-term run from %s, %s %s"
                        % (me, _mask_desc(s), s.last_written_index,
                           [s.peers[p].match_index for p in others], _run_of_term(s, T), kind,
                           "to %d" % b if kind == "written" else "from slot %d last_index %d" % (ev.from_slot, b)))
                out.append(Case("commit" if kind != "unknown" else "commit-unknown", s, ev, desc))
    return out


def _run_of_term(s, t):
    return next((s.run_start[k] for k in range(s.n_runs) if s.run_term[k] == t), None)


def vote_cases(m, rng):
    """candidates and pre-voters at every slot, every voter mask of all M slots, 0..M-1 votes already counted"""
    out = []
    for role in (abi.CANDIDATE, abi.PRE_VOTE):
        masks = _masks(m, rng, 64)
        for mask in masks * max(1, 32 // len(masks)):
            rq = required_quorum(bin(mask).count("1"))
            picks = {rng.randrange(m)} | ({rq - 1} if rq - 1 < m else set())
            for votes in sorted(picks):
                me = rng.randrange(m)
                s = _member(m, me)
                abi.set_log(s, [(i, T - 1) for i in range(1, C0 + 1)], last_written=(C0, T - 1))
                s.role, s.current_term, s.votes, s.voted_for = role, T, votes, me
                s.commit_index, s.last_applied = C0 - 2, C0 - 2
                s.membership = abi.VOTER if mask >> me & 1 else rng.choice([abi.NON_VOTER, abi.PROMOTABLE])
                s.pre_vote_token = s.token_counter = 2
                for p in range(m):
                    s.peers[p].voter = mask >> p & 1
                    s.peers[p].next_index = C0 + 1
                f = rng.choice([p for p in range(m) if p != me] or [me])
                ev = (abi.ev_request_vote_result(0, T, True, voter=f) if role == abi.CANDIDATE else
                      abi.ev_pre_vote_result(0, T, 2, True, voter=f))
                desc = "%s slot %d voters %s (quorum %d) membership %d, %d votes + 1" % (
                    abi.ROLE_NAMES[role], me, _mask_desc(s), rq, s.membership, votes)
                out.append(Case("vote", s, ev, desc))
    return out


def query_cases(m, rng, n=48):
    """leaders with their own and their peers' query indexes; one heartbeat reply from a voter, a non-voter or a
    slot outside the group"""
    out = []
    for _ in range(n):
        me = rng.randrange(m)
        others = [p for p in range(m) if p != me]
        voters = {p for p in others if rng.random() < 0.7}
        s = _leader(m, me, voters, rng, C0)
        q = abi.RaQueryState(query_index=rng.randint(1, 4), agreed_index=rng.randint(0, 3))
        for p in others:
            q.peer_query_index[p] = rng.randint(0, 4)
        f = rng.choice(others + [m, 9]) if others else m
        ev = abi.ev_heartbeat_reply(0, f, T, rng.randint(0, 5))
        desc = "leader slot %d voters %s query_index %d peers %s agreed %d, reply from slot %d index %d" % (
            me, _mask_desc(s), q.query_index, [q.peer_query_index[p] for p in others], q.agreed_index, f, ev.a)
        out.append(Case("query", s, ev, desc, q))
    return out


def table(m):
    """Every case of M members: case i is group i, its member at the case's slot is row slot * G + i."""
    rng = random.Random(1000 + m)
    cases = commit_cases(m, rng) + vote_cases(m, rng) + query_cases(m, rng)
    G = len(cases)
    for g, c in enumerate(cases):
        c.state.row = c.event.row = c.state.self_slot * G + g
        if c.query is not None:
            c.query.row = c.state.row
    return G, cases


# ---- one run --------------------------------------------------------------------------------------------------------
def _check_rule(b, m, setting, cases, pure):
    """Each case's read-back commit index, role and votes, or agreed index, against the restated rule."""
    rows = b.read_rows([c.state.row for c in cases])
    qs = b.read_query_state([c.state.row for c in cases])
    bad = []
    for c, s, q in zip(cases, rows, qs):
        base = c.state.commit_index
        if c.kind == "commit":
            want, got, what = expected_commit(s, base), s.commit_index, "commit_index"
        elif c.kind == "commit-unknown":                        # a reply from outside the cluster map is not counted
            want, got, what = base, s.commit_index, "commit_index"
        elif c.kind == "vote":
            rq = required_quorum(sum(c.state.peers[p].voter for p in range(m)))
            counted = c.state.role == abi.CANDIDATE or c.member_voter     # a pre-vote counts for a voter only
            won = counted and c.votes + 1 == rq
            if c.state.role == abi.CANDIDATE:
                role = abi.LEADER if won else abi.CANDIDATE
            else:                                               # call_for_election(candidate): its own vote is chased
                role = (abi.LEADER if rq == 1 and not pure else abi.CANDIDATE) if won else abi.PRE_VOTE
            want, got, what = role, s.role, "role"
            if s.role == role and not won:
                want, got, what = c.votes + (1 if counted else 0), s.votes, "votes"
        else:
            vq = [q.query_index] + [q.peer_query_index[p] for p in range(m)
                                    if p != s.self_slot and s.peers[p].voter]
            want, got, what = max(c.query.agreed_index, agreed_commit(vq)), q.agreed_index, "agreed_index"
        if want != got:
            bad.append("%s: expected %s %d, got %d" % (c.desc, what, want, got))
    assert not bad, "M=%d %s %s: %d of %d cases differ from the rule, e.g.\n  %s" % (
        m, setting, b.name, len(bad), len(cases), "\n  ".join(bad[:8]))


def _coverage(m, cases, oracle):
    """The table reaches what it is for: the commit index advances, is held by the §5.4.2 gate, moves back; votes
    win, fall short and overshoot the quorum."""
    rows = oracle.read_rows([c.state.row for c in cases])
    seen = set()
    for c, s in zip(cases, rows):
        if c.kind == "commit":
            idx = [s.last_written_index] + [s.peers[p].match_index for p in range(m)
                                            if p != s.self_slot and s.peers[p].voter]
            cand, base = agreed_commit(idx), c.state.commit_index
            seen.add("gate closed" if term_at(s, cand) != s.current_term and cand > base else
                     "advanced" if s.commit_index > base else "moved back" if s.commit_index < base else "held")
        elif c.kind == "vote":
            rq = required_quorum(sum(c.state.peers[p].voter for p in range(m)))
            seen.add("quorum" if c.votes + 1 == rq else "past quorum" if c.votes + 1 > rq else "short")
    want = {"advanced", "gate closed", "held", "moved back", "quorum", "short", "past quorum"}
    if m == 1:
        want -= {"short", "past quorum"}                        # one member: no vote before its own
    assert want <= seen, "M=%d: the table does not reach %s" % (m, want - seen)


def run_table(backend, setting, m, monkeypatch):
    cfg, wide, shift, hot = SETTINGS[setting]
    monkeypatch.setenv("RA_STEP_WIDE", wide)
    G, cases = table(m)
    rows, qs, events = [clone(c.state) for c in cases], [c.query for c in cases if c.query is not None], []
    for c in cases:
        e = clone(c.event)
        if shift:
            shift_event(e, *shift)
        events.append(e)
    if shift:
        for s in rows:
            shift_state(s, shift[0], shift[1], m)
        for c in cases:                                         # the rule is checked against the moved values
            shift_state(c.state, shift[0], shift[1], m)
    events.sort(key=lambda e: e.row)
    o = Oracle(G, m, **cfg)
    bs = [o] if backend == "oracle" else [o, make_backend(backend, G, m, **cfg)]
    Emu.narrow_stats()
    outs = []
    for b in bs:
        b.load_rows(rows)
        b.load_query_state(qs)
        outs.append(b.step([clone(e) for e in events]))
    ns = Emu.narrow_stats()
    b = bs[-1]
    _check_rule(b, m, setting, cases, cfg.get("pure", False))
    if backend == "oracle":
        _coverage(m, cases, o)
        return
    compare(observe(o, m, outs[0]), observe(b, m, outs[1]), "M=%d %s %s" % (m, setting, backend), events, o)
    # which kernel took the leaders' replies: a stall counts (role, event type) in the general kernel
    replies = sum(1 for c in cases if c.event.type == abi.EV_AER_REPLY)
    unknown = sum(1 for c in cases if c.kind == "commit-unknown")
    stalled = b.stall_histogram().get((abi.LEADER, abi.EV_AER_REPLY), 0)
    if cfg.get("pure"):
        assert stalled == replies, "M=%d %s: %d of %d replies took the general kernel" % (m, setting, stalled, replies)
    elif hot:                                                   # (a reply from outside the group always stalls)
        assert stalled <= unknown + replies // 50, "M=%d %s: %d of %d replies (%d from outside the group) left the " \
            "hot kernel" % (m, setting, stalled, replies, unknown)
    if backend == "emu" and m == 5 and not cfg.get("pure") and wide == "0":   # the emulation's 32-bit pass: M = 5
        if shift:                                               # every row refused to the general kernel
            assert ns["rows_narrow"] == 0 and ns["rows_wide"] >= len(cases), ns
        else:
            assert ns["rows_narrow"] >= len(cases) and ns["rows_wide"] == 0, ns


@pytest.mark.parametrize("m", MEMBERS)
@pytest.mark.parametrize("setting", list(SETTINGS))
@pytest.mark.parametrize("backend", ["oracle", "emu"])
def test_quorum_table(backend, setting, m, monkeypatch):
    run_table(backend, setting, m, monkeypatch)


@pytest.mark.gpu
@pytest.mark.parametrize("m", MEMBERS)
@pytest.mark.parametrize("setting", list(SETTINGS))
def test_quorum_table_engine(setting, m, monkeypatch):
    run_table("engine", setting, m, monkeypatch)
