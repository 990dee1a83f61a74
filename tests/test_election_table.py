"""Who leads in which term: every step kernel's term, vote and step-down clauses against the rule restated in a few lines.

raft_logic.cuh decides elections in update_term / update_term_and_voted_for, is_candidate_log_up_to_date,
process_pre_vote (term, log, protocol version, the machine-version gate, the token, whether a follower replies at all),
call_for_election for both targets, the role handlers' higher-term step-downs and {next_event, Msg} redispatches, the
leader's same-term fatals, its failed append_entries_reply back-off and handle_await_condition; the hot kernel takes a
follower's pre_vote, election timeout and ignored vote results, a pre-voter's AppendEntries at term >= current and a
leader's enforce-leadership itself (fast_event), under guards that differ in the 32-bit pass.  Here each clause is
restated once more, citing ra_server.erl as the kernels do, and for every M from 1 to 8 the table holds one crafted
member per group:

- every role x REQUEST_VOTE, REQUEST_VOTE_RES, PRE_VOTE, PRE_VOTE_RES, AER, AER_REPLY (failed, or at a higher or lower
  term), HEARTBEAT_RPC, HEARTBEAT_REPLY, ELECTION_TIMEOUT and AWAIT_COND_TIMEOUT; event terms one below, equal to and
  one above current; the candidate's log older, equal or newer by term and by index; voted_for undefined, self, the
  candidate or another slot; membership voter, promotable or non_voter; senders a voter, a non-voter, a slot M..14 or
  RA_NO_SLOT;
- pre_votes of protocol version 0, 1 and 2 with (their, ours, effective) machine versions drawn from 0..3, and pre-vote
  results whose token matches, is stale or is from the future;
- a leader's failed replies from a peer whose last index is in the log with the same term, with another term below or
  above match_index, at the snapshot index, above last_index, or from an unknown slot, over a literal {index: term} log;
- await_condition rows with the condition `missing` or `term_mismatch`, its reply valid or not, a leader or none;
- token_counter at 2^30 - 1 and 2^30, followers with machine_version != 0 timing out, pre_votes whose version word does
  not fit 32 bits, and quorums of one (M = 1, or one voter), where an election timeout reaches leader in one step.

AppendEntries here are empty with prev at the receiver's last entry (right or wrong term) or prev missing, so the
follower clause they reach is one tests/test_log_view_table.py pins; a leader's successful reply is the quorum table's.

After one step the read-back role, term, vote, leader, votes, token, peers' next / match indexes and condition, each
row's STATUS bits, the election counters and (host-routed and pure) every vote, pre-vote, AppendEntries reply and
heartbeat reply record -- and in pure mode every {next_event, _} -- must equal the rule; the emulation and the engine
must equal the oracle.  The stall histogram must equal the restated `hot_event`.  A batch with a sender slot in
15..254 is RA_E_INVAL on every backend and changes no row.
"""
import copy
import functools
import random
from collections import Counter

import pytest

from fuzz_lib import TABLE_SETTINGS as SETTINGS, compare, observe, shift_event, shift_state
from oracle_lib import Oracle
from ra_b200 import abi
from ra_suite import clone, make_backend

NO = abi.RA_NO_SLOT
UNDEF = abi.RA_UNDEF_TERM
LIM = 1 << 30
MEMBERS = list(range(1, abi.RA_MAX_MEMBERS + 1))
T = 7                                                   # current term of the crafted rows
SNAP = (2, 1)                                           # the log: a snapshot, then three term runs
LOG = {3: 2, 4: 2, 5: 4, 6: 4, 7: 4, 8: 6, 9: 6}
LAST, LT = 9, 6
COMMIT, APPLIED = 6, 5
ROLES = [abi.FOLLOWER, abi.CANDIDATE, abi.PRE_VOTE, abi.LEADER, abi.AWAIT_CONDITION]
TYPES = [abi.EV_REQUEST_VOTE, abi.EV_REQUEST_VOTE_RES, abi.EV_PRE_VOTE, abi.EV_PRE_VOTE_RES, abi.EV_AER,
         abi.EV_AER_REPLY, abi.EV_HEARTBEAT_RPC, abi.EV_HEARTBEAT_REPLY, abi.EV_ELECTION_TIMEOUT,
         abi.EV_AWAIT_COND_TIMEOUT]
# the candidate's (last_index, last_term) against ours (9, 6)
CAND_LOGS = {"equal": (LAST, LT), "older term": (LAST, LT - 1), "newer term": (4, LT + 1),
             "older index": (LAST - 1, LT), "newer index": (LAST + 1, LT)}
STATUS_BITS = (abi.ST_TERM_VOTE_CHANGED | abi.ST_ROLE_CHANGED | abi.ST_LEADER_MSG | abi.ST_START_ELECTION_TMO |
               abi.ST_BECAME_LEADER)
COUNTERS = ("elections", "pre_vote_elections", "term_and_voted_for_updates", "aer_replies_failed", "elections_won",
            "fatal_rows")
CHECKED = {abi.EV_REQUEST_VOTE, abi.EV_REQUEST_VOTE_RES, abi.EV_PRE_VOTE, abi.EV_PRE_VOTE_RES, abi.EV_AER_REPLY,
           abi.EV_HEARTBEAT_REPLY}
MAX_PIPE, MAX_BATCH = 4096, 128                         # abi.Backend's defaults


# ---- the rule, restated ---------------------------------------------------------------------------------------------
class Mem:
    """A member as ra_server keeps what this table touches: role, term, vote, leader, votes, membership, the voters,
    machine versions, the pre-vote token and counter, a literal {index: term} log with a snapshot, peers' (next, match,
    commit_index_sent), the await condition; and what one step emitted."""

    def __init__(self, m, me, role):
        self.m, self.me, self.role = m, me, role
        self.term, self.voted, self.leader, self.votes = T, NO, NO, 0
        self.membership, self.voter = abi.VOTER, [1] * m
        self.mv = self.eff = 0
        self.tok = self.ctr = 5
        self.t, self.snap, self.last, self.last_term = dict(LOG), SNAP, LAST, LT
        self.lw, self.commit, self.applied = (LAST, LT), COMMIT, APPLIED
        self.peers = [[LAST + 1, LAST, COMMIT] for _ in range(m)]
        self.cond, self.cond_valid, self.cond_reply = 0, 0, (0, 0, 0, 0)
        self.status, self.fatal = 0, 0
        self.msgs, self.nexts, self.tags, self.cnt = [], [], set(), Counter()

    def __deepcopy__(self, memo):
        x = copy.copy(self)
        x.voter, x.t, x.peers = list(self.voter), dict(self.t), [list(p) for p in self.peers]
        x.msgs, x.nexts, x.tags, x.cnt = list(self.msgs), list(self.nexts), set(self.tags), Counter(self.cnt)
        return x

    def row(self, row):
        s = abi.empty_row(row, 1, self.m)
        s.row, s.self_slot = row, self.me
        abi.set_log(s, sorted(self.t.items()), last_written=self.lw, snapshot=self.snap)
        s.role, s.current_term, s.voted_for, s.leader_slot, s.votes = self.role, self.term, self.voted, self.leader, \
            self.votes
        s.membership, s.machine_version, s.effective_machine_version = self.membership, self.mv, self.eff
        s.pre_vote_token, s.token_counter = self.tok, self.ctr
        s.commit_index, s.last_applied = self.commit, self.applied
        for p in range(self.m):
            s.peers[p].next_index, s.peers[p].match_index, s.peers[p].commit_index_sent = self.peers[p]
            s.peers[p].voter = self.voter[p]
        s.condition = self.cond
        if self.cond_valid:
            s.flags |= 2
            s.cond_reply_term, s.cond_reply_next_index, s.cond_reply_last_index, s.cond_reply_last_term = \
                self.cond_reply
        return s


def fetch_term(S, i):
    """ra_log:fetch_term/2 (ra_log.erl:1140-1152): undefined outside the log, the snapshot index included"""
    return S.t.get(i)


def srv_fetch_term(S, i):
    """fetch_term/2 :3158-3169: falls back on the snapshot"""
    t = fetch_term(S, i)
    return S.snap[1] if t is None and S.snap and S.snap[0] == i else t


def update_term_and_voted_for(S, term, voted):
    """update_term_and_voted_for/3 :3014-3031: counted, and persisted (STATUS), only when something changes"""
    if term == S.term and voted == S.voted:
        return
    S.cnt["term_and_voted_for_updates"] += 1
    S.term, S.voted = term, voted
    S.status |= abi.ST_TERM_VOTE_CHANGED


def update_term(S, term):
    """update_term/2 :3033-3037"""
    if term > S.term:
        update_term_and_voted_for(S, term, NO)


def up_to_date(idx, term, S):
    """is_candidate_log_up_to_date/3 :3132-3139"""
    return term > S.last_term or (term == S.last_term and idx >= S.last)


def required_quorum(S):
    """required_quorum/1 :3969-3972"""
    return sum(S.voter) // 2 + 1


def send(S, type_, to, term, a=0, b=0, c=0, d=0):
    S.msgs.append((type_, to, term, a, b, c, d))


def reply_vote(S, to, type_, term, token, granted, why):
    S.tags.add("%s %s: %s" % ("pre_vote" if type_ == abi.EV_PRE_VOTE_RES else "vote", "granted" if granted else
                              "declined", why))
    send(S, type_, to, term, 0, 0, token, 1 if granted else 0)


def aer_reply(S, term, ok):
    """append_entries_reply/3 :3597-3604"""
    send(S, abi.EV_AER_REPLY, S.leader, term, S.last + 1, S.lw[0], S.lw[1], 1 if ok else 0)


def call_for_election(S, target, nq):
    """call_for_election/3 :2853-2897: a new term (candidate) or a fresh token (pre_vote), voted for self, leader
    undefined, no votes, one request to every other slot, then the vote for self as a next event"""
    if target == abi.CANDIDATE:
        nt = S.term + 1
        S.cnt["elections"] += 1                                             # :2856
        req = (abi.EV_REQUEST_VOTE, nt, S.last, S.last_term, 0, 0)
        update_term_and_voted_for(S, nt, S.me)
        nq.append("self_vote")
    else:
        token = S.ctr + 1                                                   # make_ref()
        S.cnt["pre_vote_elections"] += 1                                    # :2878
        req = (abi.EV_PRE_VOTE, S.term, S.last, S.last_term, token, 1 | (S.mv << 32))
        update_term_and_voted_for(S, S.term, S.me)
        S.tok = S.ctr = token
        nq.append("self_pre_vote")
    S.leader, S.votes = NO, 0
    S.tags.add("election: " + abi.ROLE_NAMES[target])
    for s in range(S.m):
        if s != S.me:
            send(S, req[0], s, *req[1:])
    return target


def process_pre_vote(S, fsm, e):
    """process_pre_vote/3 :2899-2956"""
    term, token, version, their = e["term"], e["c"], e["d"] & 0xffffffff, e["d"] >> 32
    if term >= S.term:
        update_term(S, term)
        if up_to_date(e["a"], e["b"], S):
            if version > 1:                                                 # :2914-2917
                reply_vote(S, e["from"], abi.EV_PRE_VOTE_RES, term, token, False, "protocol version")
            elif their == S.eff or S.eff <= their <= S.mv:                  # :2918-2928
                reply_vote(S, e["from"], abi.EV_PRE_VOTE_RES, term, token, True,
                           "machine version equal" if their == S.eff else "machine version in range")
            else:                                                           # :2929-2934
                S.status |= abi.ST_START_ELECTION_TMO
                reply_vote(S, e["from"], abi.EV_PRE_VOTE_RES, term, token, False,
                           "machine version above ours" if their > S.mv else "machine version below effective")
        elif fsm == abi.FOLLOWER:                                           # :2941-2942: no reply
            S.status |= abi.ST_START_ELECTION_TMO
            S.tags.add("pre_vote declined: follower stays silent")
        else:                                                               # :2943-2945
            reply_vote(S, e["from"], abi.EV_PRE_VOTE_RES, term, token, False, "log behind")
    else:                                                                   # :2948-2956
        reply_vote(S, e["from"], abi.EV_PRE_VOTE_RES, S.term, token, False, "lower term")
    return fsm


def has_entry(S, idx, term):
    """has_log_entry_or_snapshot/3 :3141-3156"""
    t = fetch_term(S, idx)
    if t is None:
        if S.snap and S.snap[0] == idx:
            return "ok" if S.snap[1] == term else "term_mismatch"
        return "missing"
    return "ok" if t == term else "term_mismatch"


def follower(S, e, nq):
    """handle_follower/2 :1264-1641, the clauses this table reaches"""
    ty = e["type"]
    if ty == abi.EV_AER:                                                    # :1266-1424, empty AppendEntries only
        if e["term"] < S.term:                                              # :1415-1424
            S.tags.add("AppendEntries at a lower term")
            send(S, abi.EV_AER_REPLY, e["from"], S.term, S.last + 1, S.lw[0], S.lw[1], 0)
            return abi.FOLLOWER
        S.status |= abi.ST_LEADER_MSG
        S.leader = e["from"]
        update_term(S, e["term"])
        r = has_entry(S, e["a"], e["b"])
        S.tags.add("AppendEntries prev " + r)
        if r == "ok":                                                       # prev == last_index: validated :1313-1326
            S.commit = e["c"]
            aer_reply(S, e["term"], True)
            return abi.FOLLOWER
        if r == "missing":                                                  # :1373-1387
            aer_reply(S, e["term"], False)
            S.cond, S.cond_valid, S.cond_reply = 1, 1, S.msgs[-1][2:6]
            return abi.AWAIT_CONDITION
        la, lat = S.applied, srv_fetch_term(S, S.applied)                   # :1388-1413, :3587-3595
        send(S, abi.EV_AER_REPLY, S.leader, e["term"], la + 1, la, lat, 0)
        S.cond, S.cond_valid, S.cond_reply = 2, 1, S.msgs[-1][2:6]
        return abi.AWAIT_CONDITION
    if ty == abi.EV_PRE_VOTE:                                               # :1459-1466
        if S.membership != abi.VOTER:
            S.tags.add("pre_vote ignored: not a voter")
            return abi.FOLLOWER
        return process_pre_vote(S, abi.FOLLOWER, e)
    if ty == abi.EV_REQUEST_VOTE:                                           # :1467-1513
        cand = e["from"]
        if S.membership != abi.VOTER:
            S.tags.add("vote ignored: not a voter")
            return abi.FOLLOWER
        if e["term"] == S.term and S.voted not in (NO, cand):
            reply_vote(S, cand, abi.EV_REQUEST_VOTE_RES, e["term"], 0, False, "already voted")
        elif e["term"] >= S.term:
            update_term(S, e["term"])
            if up_to_date(e["a"], e["b"], S):
                reply_vote(S, cand, abi.EV_REQUEST_VOTE_RES, e["term"], 0, True, "log up to date")
                update_term_and_voted_for(S, e["term"], cand)
            else:
                reply_vote(S, cand, abi.EV_REQUEST_VOTE_RES, e["term"], 0, False, "log behind")
        else:
            reply_vote(S, cand, abi.EV_REQUEST_VOTE_RES, S.term, 0, False, "lower term")
        return abi.FOLLOWER
    if ty in (abi.EV_AER_REPLY, abi.EV_HEARTBEAT_REPLY):                     # :1514-1521
        update_term(S, e["term"])
        return abi.FOLLOWER
    if ty == abi.EV_ELECTION_TIMEOUT:                                       # :1603-1610
        if S.membership != abi.VOTER:
            S.tags.add("election timeout ignored: not a voter")
            return abi.FOLLOWER
        return call_for_election(S, abi.PRE_VOTE, nq)
    if ty == abi.EV_HEARTBEAT_RPC:                                          # :1425-1440
        if e["term"] >= S.term:
            update_term(S, e["term"])
            S.leader = e["from"]
            send(S, abi.EV_HEARTBEAT_REPLY, e["from"], e["term"], e["a"])
        else:
            send(S, abi.EV_HEARTBEAT_REPLY, e["from"], S.term, e["a"])
        return abi.FOLLOWER
    return abi.FOLLOWER                                                     # vote results :1593-1598, ...


def make_aer(S, prev, num):
    """make_append_entries_rpc/6 :2401-2418, cut after its second term run (DESIGN §2 item 2): the new next_index"""
    frm, to = prev + 1, min(S.last, prev + num)
    if to >= frm and fetch_term(S, frm) is not None:
        i, d = frm, fetch_term(S, frm)
        while i <= to and fetch_term(S, i) == d:
            i += 1
        if i <= to:
            j, x = i, fetch_term(S, i)
            while j <= to and fetch_term(S, j) == x:
                j += 1
            to = j - 1
    else:
        to = min(frm - 1, S.last)
    return to + 1


def pipeline_pass(S, pure, force=False):
    """make_pipelined_rpc_effects/3 :2268-2329 with make_rpc_effect/5 :2365-2399 (the records are not checked here:
    only where each peer's next_index ends up)"""
    for s in range(S.m):
        if s == S.me:
            continue
        nx, mt, cs = S.peers[s]
        if not (nx < S.last + 1 or cs < S.commit):
            continue
        inflight = nx - mt - 1
        if not (inflight < MAX_PIPE or force):
            continue
        bs = max(1, min(MAX_PIPE - inflight, MAX_BATCH))
        prev = nx - 1
        if fetch_term(S, prev) is not None or prev == S.snap[0]:
            nn = make_aer(S, prev, bs)
            S.tags.add("AppendEntries from the snapshot" if prev == S.snap[0] else "AppendEntries from the log")
        elif prev < S.snap[0]:
            S.tags.add("snapshot sent")
            nn = S.snap[0]
        else:
            S.fatal = abi.FATAL_ASSERT
            return
        S.peers[s] = [nn, mt, S.commit]


def step_down(S, term):
    """the leader's {next_event, Msg} on a higher term: leader undefined, update_term/2"""
    S.leader = NO
    update_term(S, term)
    return abi.FOLLOWER


def leader(S, e, nq, pure):
    """handle_leader/2 :520-1023, the clauses this table reaches"""
    ty, known = e["type"], e["from"] < S.m
    if ty == abi.EV_AER_REPLY:
        ok = e["d"] != 0
        if e["term"] > S.term:                                              # :562-576
            if not known:
                S.tags.add("higher-term reply from an unknown slot ignored")
                return abi.LEADER
            S.tags.add("step down: reply")
            return step_down(S, e["term"])
        if not ok:                                                          # :577-643
            if not known:
                S.tags.add("back-off: unknown slot")
                return abi.LEADER
            S.cnt["aer_replies_failed"] += 1
            nx, mt, cs = S.peers[e["from"]]
            pnext, plast, plt = e["a"], e["b"], e["c"]
            t = fetch_term(S, plast)
            if t is None:
                nn = pnext
                S.tags.add("back-off: last index not found")
            elif t == plt and plast >= mt:
                mt, nn = plast, pnext
                S.tags.add("back-off: same term")
            elif plast < mt:
                mt, nn = plast, plast + 1
                S.tags.add("back-off: below match_index")
            else:
                nn = max(min(nx - 1, pnext), mt)
                S.tags.add("back-off: other term above match_index")
            S.peers[e["from"]] = [nn, mt, cs]
            pipeline_pass(S, pure)
        return abi.LEADER
    if ty == abi.EV_AER:
        if e["term"] > S.term:                                              # :826-835
            S.tags.add("step down: AppendEntries")
            nq.append("redispatch")
            return step_down(S, e["term"])
        if e["term"] == S.term:                                             # :836-840
            S.fatal = abi.FATAL_LEADER_SAW_AER_SAME_TERM
            S.tags.add("fatal: AppendEntries in the same term")
            return abi.LEADER
        send(S, abi.EV_AER_REPLY, e["from"], S.term, S.last + 1, S.lw[0], S.lw[1], 0)   # :841-845
        return abi.LEADER
    if ty in (abi.EV_REQUEST_VOTE, abi.EV_PRE_VOTE):
        if e["term"] > S.term:                                              # :919-951
            if not known:
                S.tags.add("higher-term request from an unknown slot ignored")
                return abi.LEADER
            S.tags.add("step down: " + ("request_vote" if ty == abi.EV_REQUEST_VOTE else "pre_vote"))
            nq.append("redispatch")
            return step_down(S, e["term"])
        if ty == abi.EV_REQUEST_VOTE:                                       # :934-936
            reply_vote(S, e["from"], abi.EV_REQUEST_VOTE_RES, S.term, 0, False, "leader")
        else:
            S.tags.add("enforce leadership")                                # :952-957 (AppendEntries to every peer)
        return abi.LEADER
    if ty == abi.EV_HEARTBEAT_RPC:
        if e["term"] > S.term:                                              # :871-880
            S.tags.add("step down: heartbeat")
            nq.append("redispatch")
            return step_down(S, e["term"])
        if e["term"] < S.term:                                              # :881-888
            send(S, abi.EV_HEARTBEAT_REPLY, e["from"], S.term, e["a"])
            return abi.LEADER
        S.fatal = abi.FATAL_LEADER_SAW_HEARTBEAT_SAME_TERM                  # :889-894
        S.tags.add("fatal: heartbeat in the same term")
        return abi.LEADER
    if ty == abi.EV_HEARTBEAT_REPLY and e["term"] > S.term:                 # :895-918
        return step_down(S, e["term"])
    return abi.LEADER


def candidate(S, e, nq):
    """handle_candidate/2 :1026-1171"""
    ty = e["type"]
    if ty == abi.EV_REQUEST_VOTE_RES:
        if e["d"] and e["term"] == S.term:                                  # :1028-1044
            nv = S.votes + 1
            if nv == required_quorum(S):
                S.leader, S.votes = S.me, 0
                for s in range(S.m):                                        # initialise_peers/1 :3207-3215
                    S.peers[s] = [S.last + 1, 0, 0]
                S.cnt["elections_won"] += 1
                S.tags.add("candidate wins")
                nq.append("noop")
                return abi.LEADER
            S.votes = nv
            return abi.CANDIDATE
        if e["term"] > S.term:                                              # :1045-1052
            update_term_and_voted_for(S, e["term"], NO)
            return abi.FOLLOWER
        return abi.CANDIDATE
    if ty in (abi.EV_AER, abi.EV_HEARTBEAT_RPC):                             # :1055-1058, :1064-1067
        if e["term"] >= S.term:
            update_term_and_voted_for(S, e["term"], NO)
            nq.append("redispatch")
            return abi.FOLLOWER
        if ty == abi.EV_AER:                                                # :1059-1063
            send(S, abi.EV_AER_REPLY, e["from"], S.term, S.last + 1, S.lw[0], S.lw[1], 0)
        else:                                                               # :1068-1073
            send(S, abi.EV_HEARTBEAT_REPLY, e["from"], S.term, e["a"])
        return abi.CANDIDATE
    if ty in (abi.EV_AER_REPLY, abi.EV_HEARTBEAT_REPLY):                     # :1082-1090, :1074-1081
        if e["term"] > S.term:
            update_term_and_voted_for(S, e["term"], NO)
            return abi.FOLLOWER
        return abi.CANDIDATE
    if ty in (abi.EV_REQUEST_VOTE, abi.EV_PRE_VOTE):
        if e["term"] > S.term:                                              # :1091-1106
            update_term_and_voted_for(S, e["term"], NO)
            nq.append("redispatch")
            return abi.FOLLOWER
        if ty == abi.EV_REQUEST_VOTE:                                       # :1107-1109
            reply_vote(S, e["from"], abi.EV_REQUEST_VOTE_RES, S.term, 0, False, "candidate")
            return abi.CANDIDATE
        return process_pre_vote(S, abi.CANDIDATE, e)                        # :1110-1114
    if ty == abi.EV_ELECTION_TIMEOUT:
        return call_for_election(S, abi.CANDIDATE, nq)
    return abi.CANDIDATE


def pre_vote(S, e, nq):
    """handle_pre_vote/2 :1173-1261"""
    ty = e["type"]
    if ty in (abi.EV_AER, abi.EV_HEARTBEAT_RPC, abi.EV_REQUEST_VOTE):
        higher = e["term"] > S.term if ty == abi.EV_REQUEST_VOTE else e["term"] >= S.term
        if higher:                                                          # :1175-1186, :1196-1201
            update_term(S, e["term"])
            S.votes = 0
            nq.append("redispatch")
            return abi.FOLLOWER
        if ty == abi.EV_HEARTBEAT_RPC:                                      # :1187-1191
            send(S, abi.EV_HEARTBEAT_REPLY, e["from"], S.term, e["a"])
        return abi.PRE_VOTE
    if ty == abi.EV_PRE_VOTE_RES:
        if e["term"] > S.term:                                              # :1202-1207
            update_term(S, e["term"])
            S.votes = 0
            return abi.FOLLOWER
        if e["d"] and e["term"] == S.term and e["c"] == S.tok and S.membership == abi.VOTER:   # :1212-1229
            nv = S.votes + 1
            S.tags.add("pre_vote counted")
            if nv == required_quorum(S):
                S.tags.add("pre_vote wins")
                return call_for_election(S, abi.CANDIDATE, nq)
            S.votes = nv
        elif e["d"] and e["term"] == S.term:
            S.tags.add("pre_vote not counted: " + ("token" if e["c"] != S.tok else "not a voter"))
        return abi.PRE_VOTE
    if ty == abi.EV_PRE_VOTE:
        return process_pre_vote(S, abi.PRE_VOTE, e)
    if ty == abi.EV_ELECTION_TIMEOUT:
        return call_for_election(S, abi.PRE_VOTE, nq)
    if ty == abi.EV_HEARTBEAT_REPLY and e["term"] > S.term:                 # :1192-1195
        S.votes = 0
        update_term(S, e["term"])
        return abi.FOLLOWER
    return abi.PRE_VOTE


def await_condition(S, e, nq):
    """handle_await_condition/2 :1900-1941"""
    ty = e["type"]
    if ty == abi.EV_REQUEST_VOTE:                                           # :1902-1903
        nq.append("redispatch")
        return abi.FOLLOWER
    if ty == abi.EV_PRE_VOTE:                                               # :1904-1905
        return process_pre_vote(S, abi.AWAIT_CONDITION, e)
    if ty == abi.EV_ELECTION_TIMEOUT:                                       # :1906-1913
        if S.membership != abi.VOTER:
            return abi.AWAIT_CONDITION
        return call_for_election(S, abi.PRE_VOTE, nq)
    if ty == abi.EV_AWAIT_COND_TIMEOUT:                                     # :1914-1927
        if S.cond_valid and S.leader != NO:
            S.tags.add("condition timeout: reply resent")
            send(S, abi.EV_AER_REPLY, S.leader, *S.cond_reply, 0)
            S.status |= abi.ST_LEADER_MSG
        else:
            S.tags.add("condition timeout: nothing to resend")
        S.cond, S.cond_valid = 0, 0
        return abi.FOLLOWER
    if ty == abi.EV_AER:                                                    # :1932-1941 with :2184-2202
        r = has_entry(S, e["a"], e["b"]) if e["term"] >= S.term else None
        if r == "ok" or (r == "term_mismatch" and S.cond == 1):
            S.tags.add("condition met: " + r)
            S.cond, S.cond_valid = 0, 0
            nq.append("redispatch")
            return abi.FOLLOWER
        S.tags.add("condition not met")
        return abi.AWAIT_CONDITION
    return abi.AWAIT_CONDITION                                              # heartbeats and replies dropped :1938-1940


def synth(S, code, e):
    """the event behind a next-event code (raft_logic.cuh synth_event)"""
    if code == "redispatch":
        return e
    if code == "self_pre_vote":
        return dict(type=abi.EV_PRE_VOTE_RES, term=S.term, c=S.tok, d=1, a=0, b=0, **{"from": S.me})
    if code == "self_vote":
        return dict(type=abi.EV_REQUEST_VOTE_RES, term=S.term, c=0, d=1, a=0, b=0, **{"from": S.me})
    return dict(type=abi.EV_COMMAND if code == "noop" else abi.EV_TICK, term=0, a=0, b=0, c=0, d=0, **{"from": NO})


def leader_synthetic(S, e, pure):
    """the leader's own next events after an election: tick (make_rpcs/1 over stale peers: no state moves) and the
    noop command (append_log_leader, then a forced pipeline pass)"""
    if e["type"] == abi.EV_COMMAND:
        S.last += 1
        S.t[S.last] = S.last_term = S.term
        pipeline_pass(S, pure, force=True)


def run(S, ev, pure):
    """one event through the member as ra_server_proc chases it: routed and host-routed chase every next event
    (new ones go first, a candidate that wins ticks before its noop); pure returns them as EVF_NEXT_EVENT records"""
    queue = [("redispatch", ev)]
    while queue and not S.fatal:
        code, src = queue.pop(0)
        e = synth(S, code, src)
        old, nq = S.role, []
        if old == abi.LEADER and e["type"] in (abi.EV_COMMAND, abi.EV_TICK):
            leader_synthetic(S, e, pure)
            new = old
        else:
            new = {abi.FOLLOWER: follower, abi.CANDIDATE: candidate, abi.PRE_VOTE: pre_vote,
                   abi.AWAIT_CONDITION: await_condition}[old](S, e, nq) if old != abi.LEADER else leader(S, e, nq, pure)
        if S.fatal:
            break
        if new != old:
            S.role = new
            S.status |= abi.ST_ROLE_CHANGED | (abi.ST_BECAME_LEADER if new == abi.LEADER else 0)
            if code == "redispatch" and old != abi.FOLLOWER and "redispatch" in nq:
                S.tags.add("redispatch from " + abi.ROLE_NAMES[old])
        if pure:
            S.nexts += [(x, synth(S, x, e)) for x in nq]
            continue
        front = nq if not (new == abi.LEADER and old == abi.CANDIDATE) else ["tick"] + nq
        queue = [(x, e) for x in front] + queue
    if S.fatal:
        S.cnt["fatal_rows"] += 1


def narrow_row(S):
    """does the row reach 2^30 anywhere (raft_row.cuh row_state_is_wide)?  The 32-bit pass hands such a row to the
    general kernel whole, without counting a stall"""
    return max([S.term, S.tok, S.ctr, S.last, S.commit] + [x for p in S.peers for x in p[:2]]) >= LIM


def hot_event(S, e, narrow, pure):
    """The (role, event type) under which an event leaves the hot kernel, None if fast_event takes it (or the row
    never enters the hot kernel).  fast_event (the end of raft_logic.cuh): a follower's pre_vote, ignored vote results,
    its election timeout while it is a voter, the quorum is more than one and (32-bit pass) its machine version is 0 and
    the next token fits; a same-term empty AppendEntries at its last entry; a leader's ignored vote results and its
    enforce-leadership on a pre_vote of at most its term with every peer normal and no query in flight.  A pre-voter's
    AppendEntries at term >= current runs the pre_vote clause (:1175-1180) in the hot kernel first: the row is a
    follower from there on, so when the follower fast path then refuses the rpc the stall is counted under
    (FOLLOWER, AER), not (PRE_VOTE, AER).  The 32-bit pass refuses a record with a field at or above 2^30 (the
    pre_vote's version | machine_version << 32 among them) before any of this, under the row's role."""
    ty = e["type"]
    if narrow and narrow_row(S):
        return None
    if pure:
        return (S.role, ty)
    if narrow and max(e["term"], e["a"], e["b"], e["c"], e["d"]) >= LIM:
        return (S.role, ty)
    role, term = S.role, S.term
    if role == abi.PRE_VOTE and ty == abi.EV_AER and e["term"] >= term:
        role, term = abi.FOLLOWER, e["term"]
    if role == abi.FOLLOWER:
        if ty == abi.EV_AER:
            hot = e["term"] == term and e["a"] == S.last and e["b"] == S.last_term
        elif ty == abi.EV_ELECTION_TIMEOUT:
            hot = S.membership == abi.VOTER and required_quorum(S) != 1 and not (narrow and (S.mv or S.ctr >= LIM))
        else:
            hot = ty in (abi.EV_PRE_VOTE, abi.EV_PRE_VOTE_RES, abi.EV_REQUEST_VOTE_RES)
    elif role == abi.LEADER:
        hot = ty in (abi.EV_PRE_VOTE_RES, abi.EV_REQUEST_VOTE_RES) or (ty == abi.EV_PRE_VOTE and e["term"] <= term)
    else:
        hot = False
    return None if hot else (role, ty)


# ---- the cases ------------------------------------------------------------------------------------------------------
class Case:
    def __init__(self, S, ev, desc):
        self.S, self.ev, self.desc = S, ev, desc


def ev_dict(type_, frm=NO, term=0, a=0, b=0, c=0, d=0):
    return dict(type=type_, term=term, a=a, b=b, c=c, d=d, **{"from": frm})


def to_event(row, e):
    x = abi.RaEvent(row=row, type=e["type"], from_slot=e["from"], term=e["term"], a=e["a"], b=e["b"], c=e["c"],
                    d=e["d"])
    return x


def senders(rng, S):
    """a voter, a non-voter, a slot M..14 or RA_NO_SLOT"""
    others = [p for p in range(S.m) if p != S.me]
    kinds = {"unknown slot": rng.choice([S.m, 14]), "RA_NO_SLOT": NO}
    for p in others:
        kinds.setdefault("voter" if S.voter[p] else "non-voter", p)
    return kinds


def member(rng, m, role, single_voter=False):
    me = rng.randrange(m)
    S = Mem(m, me, role)
    S.membership = rng.choice([abi.VOTER] * 4 + [abi.PROMOTABLE, abi.NON_VOTER])
    for p in range(m):
        S.voter[p] = (1 if S.membership == abi.VOTER else 0) if p == me else \
            (0 if single_voter else (1 if rng.random() < 0.75 else 0))
    S.voted = rng.choice([NO, me] + ([rng.choice([p for p in range(m) if p != me])] if m > 1 else []) + [min(m, 14)])
    if role == abi.LEADER:
        S.leader, S.voted = me, me
        S.membership, S.voter[me] = abi.VOTER, 1
    elif role in (abi.CANDIDATE, abi.PRE_VOTE):
        S.voted = me
        S.votes = rng.randint(0, max(0, required_quorum(S) - 1))
    else:
        S.leader = rng.choice([NO, min(m, 14)] + [p for p in range(m) if p != me])
    if rng.random() < 0.4:
        S.mv = rng.randint(0, 3)
        S.eff = rng.randint(0, S.mv)
    if role == abi.AWAIT_CONDITION:
        S.cond = rng.choice([1, 2])
        S.cond_valid = rng.choice([0, 1, 1])
        S.cond_reply = (T, LAST + 1, LAST, LT) if S.cond == 1 else (T, APPLIED + 1, APPLIED, LOG[APPLIED])
    return S


def event_for(rng, S, ty):
    """one event of type ty for S, with a description"""
    dt = rng.choice([-1, 0, 1])
    term = S.term + dt
    snd = senders(rng, S)
    kind = rng.choice(sorted(snd))
    f = snd[kind]
    what = "term %+d from %s" % (dt, kind)
    if ty in (abi.EV_REQUEST_VOTE, abi.EV_PRE_VOTE):
        if S.voted not in (NO, S.me) and ty == abi.EV_REQUEST_VOTE and rng.random() < 0.3:
            f = S.voted                                                     # the one it voted for asks again
            what = "term %+d from the slot voted for" % dt
        lk = rng.choice(sorted(CAND_LOGS))
        a, b = CAND_LOGS[lk]
        what += ", log %s" % lk
        if ty == abi.EV_REQUEST_VOTE:
            return ev_dict(ty, f, term, a, b), what
        version, their = rng.choice([0, 1, 1, 2]), rng.randint(0, 3)
        token = rng.randint(1, 9)
        return ev_dict(ty, f, term, a, b, token, version | (their << 32)), what + ", version %d machine %d" % (
            version, their)
    if ty in (abi.EV_REQUEST_VOTE_RES, abi.EV_PRE_VOTE_RES):
        granted = rng.random() < 0.8
        tk = rng.choice(["match", "match", "stale", "future"])
        token = {"match": S.tok, "stale": S.tok - 1, "future": S.tok + 1}[tk] if ty == abi.EV_PRE_VOTE_RES else 0
        return ev_dict(ty, f, term, 0, 0, token, 1 if granted else 0), what + (", %s token" % tk if token else "") + \
            (" granted" if granted else " declined")
    if ty == abi.EV_AER:
        ak = rng.choice(["at last", "at last", "wrong term", "missing"])
        prev, pt = {"at last": (LAST, LT), "wrong term": (LAST, LT - 1), "missing": (LAST + 2, LT)}[ak]
        return ev_dict(ty, f, term, prev, pt, COMMIT), what + ", prev " + ak
    if ty == abi.EV_AER_REPLY:
        if S.role == abi.LEADER and dt <= 0:
            return backoff_event(rng, S, f, term), what + ", failed"
        ok = rng.random() < 0.3 and dt != 0
        return ev_dict(ty, f, term, LAST + 1, LAST, LT, 1 if ok else 0), what
    if ty in (abi.EV_HEARTBEAT_RPC, abi.EV_HEARTBEAT_REPLY):
        return ev_dict(ty, f, term, rng.randint(1, 4)), what
    return ev_dict(ty), "host event"


def backoff_event(rng, S, f, term):
    """a failed reply: the peer's last index in the log with the same term, with another term, at the snapshot,
    below it or above last_index; its match / next somewhere below"""
    if f < S.m:
        mt = rng.randint(2, LAST)
        S.peers[f] = [rng.randint(mt + 1, LAST + 1), mt, COMMIT]
    plast = rng.choice([SNAP[0] - 1, SNAP[0], 3, 4, 5, 6, 7, 8, 9, LAST + 1, LAST + 3])
    right = fetch_term(S, plast)
    plt = right if right is not None and rng.random() < 0.5 else rng.choice([1, 3, 5, LT])
    return ev_dict(abi.EV_AER_REPLY, f, term, plast + 1, plast, plt, 0)


def table_cases(rng, m):
    out = []
    for role in ROLES:
        for ty in TYPES:
            for _ in range(14 if ty in (abi.EV_REQUEST_VOTE, abi.EV_PRE_VOTE, abi.EV_AER_REPLY) else 8):
                S = member(rng, m, role)
                ev, what = event_for(rng, S, ty)
                out.append(Case(S, ev, "%s slot %d %s votes %d voted %s membership %d mv %d/%d: %s" % (
                    abi.ROLE_NAMES[role], S.me, "".join("V" if v else "-" for v in S.voter), S.votes, S.voted,
                    S.membership, S.mv, S.eff, what)))
    # every back-off branch: the peer's last index at each place in the log, its term right or wrong, match_index
    # below or above it; and each higher-term request from a peer that steps the leader down
    if m > 1:
        for plast in (SNAP[0] - 1, SNAP[0], 3, 4, 5, 6, 7, 8, 9, LAST + 1, LAST + 3):
            for right in (True, False):
                S = member(rng, m, abi.LEADER)
                f = rng.choice([p for p in range(m) if p != S.me])
                mt = rng.randint(2, LAST)
                S.peers[f] = [rng.randint(mt + 1, LAST + 1), mt, COMMIT]
                plt = fetch_term(S, plast) if right and fetch_term(S, plast) is not None else LT + 1
                out.append(Case(S, ev_dict(abi.EV_AER_REPLY, f, T, plast + 1, plast, plt, 0),
                                "leader: failed reply last %d term %d, match %d" % (plast, plt, mt)))
        for ty in (abi.EV_REQUEST_VOTE, abi.EV_PRE_VOTE, abi.EV_HEARTBEAT_RPC, abi.EV_AER, abi.EV_AER_REPLY):
            S = member(rng, m, abi.LEADER)
            f = rng.choice([p for p in range(m) if p != S.me])
            out.append(Case(S, ev_dict(ty, f, T + 1, LAST, LT, 1 if ty == abi.EV_PRE_VOTE else 0,
                                       1 if ty == abi.EV_PRE_VOTE else 0), "leader: higher term from slot %d" % f))
    # the leader's same-term fatals
    for ty in (abi.EV_AER, abi.EV_HEARTBEAT_RPC):
        S = member(rng, m, abi.LEADER)
        f = rng.choice(list(senders(rng, S).values()))
        out.append(Case(S, ev_dict(ty, f, T, LAST, LT), "leader: same term from slot %d" % f))
    # pre-vote results whose token matches, is stale or is from the future
    for tk in (-1, 0, 1):
        S = member(rng, m, abi.PRE_VOTE)
        S.membership, S.voter[S.me] = abi.VOTER, 1
        f = rng.choice(list(senders(rng, S).values()))
        out.append(Case(S, ev_dict(abi.EV_PRE_VOTE_RES, f, T, 0, 0, S.tok + tk, 1), "pre_vote result token %+d" % tk))
    S = member(rng, m, abi.PRE_VOTE)
    S.membership, S.voter[S.me] = abi.PROMOTABLE, 0
    out.append(Case(S, ev_dict(abi.EV_PRE_VOTE_RES, NO, T, 0, 0, S.tok, 1), "promotable pre-voter: pre_vote result"))
    # every arm of the machine-version gate :2914-2934: (their, ours, effective) in 0..3, an up-to-date log
    for mv in range(4):
        for eff in range(mv + 1):
            for their in range(4):
                S = member(rng, m, rng.choice([abi.FOLLOWER, abi.CANDIDATE, abi.PRE_VOTE, abi.AWAIT_CONDITION]))
                S.membership, S.voter[S.me], S.mv, S.eff = abi.VOTER, 1, mv, eff
                f = rng.choice(list(senders(rng, S).values()))
                out.append(Case(S, ev_dict(abi.EV_PRE_VOTE, f, T, LAST, LT, 4, rng.choice([0, 1]) | (their << 32)),
                                "%s machine versions %d/%d: pre_vote from machine version %d" % (
                                    abi.ROLE_NAMES[S.role], mv, eff, their)))
    # await_condition: either condition against each AppendEntries, the condition timeout with a leader or none
    for cond in (1, 2):
        for valid in (0, 1):
            for ak, (prev, pt) in (("at last", (LAST, LT)), ("wrong term", (LAST, LT - 1)), ("missing", (LAST + 2, LT))):
                S = member(rng, m, abi.AWAIT_CONDITION)
                S.cond, S.cond_valid = cond, valid
                f = rng.choice(list(senders(rng, S).values()))
                out.append(Case(S, ev_dict(abi.EV_AER, f, T, prev, pt, COMMIT), "condition %d valid %d: prev %s" %
                                (cond, valid, ak)))
            for ld in (NO, min(m, 14)) + ((1,) if m > 1 else ()):
                S = member(rng, m, abi.AWAIT_CONDITION)
                S.cond, S.cond_valid, S.leader = cond, valid, ld if ld != S.me else NO
                out.append(Case(S, ev_dict(abi.EV_AWAIT_COND_TIMEOUT), "condition %d valid %d leader %s: timeout" %
                                (cond, valid, S.leader)))
    # a pre-voter's vote that reaches its quorum, at every voter count
    for _ in range(6):
        S = member(rng, m, abi.PRE_VOTE)
        S.membership, S.voter[S.me] = abi.VOTER, 1
        S.votes = required_quorum(S) - 1
        out.append(Case(S, ev_dict(abi.EV_PRE_VOTE_RES, rng.choice(list(senders(rng, S).values())), T, 0, 0, S.tok, 1),
                        "pre_vote at quorum - 1"))
    # tokens at the 32-bit pass's edge, followers with a machine version timing out, pre_votes whose version word
    # does not fit 32 bits
    for ctr in (LIM - 1, LIM):
        for role in (abi.FOLLOWER, abi.PRE_VOTE, abi.AWAIT_CONDITION, abi.CANDIDATE):
            S = member(rng, m, role)
            S.tok = S.ctr = ctr
            out.append(Case(S, ev_dict(abi.EV_ELECTION_TIMEOUT), "token_counter %d: election timeout" % ctr))
            if role == abi.PRE_VOTE:
                S = member(rng, m, role)
                S.tok = S.ctr = ctr
                S.membership, S.voter[S.me] = abi.VOTER, 1
                out.append(Case(S, ev_dict(abi.EV_PRE_VOTE_RES, NO, T, 0, 0, ctr, 1), "token %d: pre_vote result" % ctr))
    for mv in (1, 2, 3):
        S = member(rng, m, abi.FOLLOWER)
        S.membership, S.voter[S.me], S.mv, S.eff = abi.VOTER, 1, mv, rng.randint(0, mv)
        out.append(Case(S, ev_dict(abi.EV_ELECTION_TIMEOUT), "follower machine version %d: election timeout" % mv))
        for role in (abi.FOLLOWER, abi.LEADER):
            S = member(rng, m, role)
            f = next(iter(senders(rng, S).values()))
            out.append(Case(S, ev_dict(abi.EV_PRE_VOTE, f, T, LAST, LT, 3, 1 | (mv << 32)),
                            "%s: pre_vote with machine version %d" % (abi.ROLE_NAMES[role], mv)))
    # a quorum of one: pre_vote -> candidate -> leader in one election timeout
    for role in (abi.FOLLOWER, abi.PRE_VOTE, abi.AWAIT_CONDITION):
        S = member(rng, m, role, single_voter=True)
        S.membership, S.voter[S.me] = abi.VOTER, 1
        out.append(Case(S, ev_dict(abi.EV_ELECTION_TIMEOUT), "%s, the only voter: election timeout" %
                        abi.ROLE_NAMES[role]))
    return out


@functools.lru_cache(maxsize=None)
def table(m):
    """Every case of M members: case i is group i, its member at the case's slot is row slot * G + i."""
    rng = random.Random(5000 + m)
    cases = table_cases(rng, m)
    return len(cases), cases


def expect(cases, pure):
    out = []
    for c in cases:
        S = copy.deepcopy(c.S)
        run(S, c.ev, pure)
        out.append(S)
    return out


# ---- one run --------------------------------------------------------------------------------------------------------
def _un(v, d):
    return v if v == UNDEF else v - d


def msg_view(x, G, di, dt):
    t = x.type
    if t == abi.EV_REQUEST_VOTE:
        return (t, x.row // G, x.term - dt, x.a - di, x.b - dt, 0, 0)
    if t == abi.EV_PRE_VOTE:
        return (t, x.row // G, x.term - dt, x.a - di, x.b - dt, x.c, x.d)
    if t in (abi.EV_REQUEST_VOTE_RES, abi.EV_PRE_VOTE_RES):
        return (t, x.row // G, x.term - dt, 0, 0, x.c, x.d)
    if t == abi.EV_AER_REPLY:
        return (t, x.row // G, x.term - dt, x.a - di, x.b - di, _un(x.c, dt), x.d)
    return (t, x.row // G, x.term - dt, x.a, 0, 0, 0)


def next_view(x, dt):
    return (x.type, x.from_slot, x.term - dt if x.type not in (abi.EV_COMMAND, abi.EV_TICK) else 0)


def model_next(code, e):
    return (e["type"], e["from"], e["term"])


def row_view(s, di, dt):
    v = dict(role=s.role, term=s.current_term - dt, voted=s.voted_for, leader=s.leader_slot, votes=s.votes,
             token=(s.pre_vote_token, s.token_counter), cond=(s.condition if s.flags & 2 else 0, (s.flags >> 1) & 1),
             peers=[(s.peers[p].next_index - di, s.peers[p].match_index and s.peers[p].match_index - di)
                    for p in range(s.n_members)])                 # (a new leader's match indexes are a plain 0)
    if s.flags & 2:
        v["cond_reply"] = (s.cond_reply_term - dt, s.cond_reply_next_index - di, s.cond_reply_last_index - di,
                           s.cond_reply_last_term - dt)
    return v


def model_view(S):
    v = dict(role=S.role, term=S.term, voted=S.voted, leader=S.leader, votes=S.votes, token=(S.tok, S.ctr),
             cond=(S.cond if S.cond_valid else 0, S.cond_valid), peers=[tuple(p[:2]) for p in S.peers])
    if S.cond_valid:
        v["cond_reply"] = tuple(S.cond_reply)
    return v


def _check_rule(b, m, setting, G, cases, want, outs, records, pure, di, dt):
    rows = b.read_rows([c.S.me * G + g for g, c in enumerate(cases)])
    msgs, notes = outs
    by_row, sent, nexts = {}, {}, {}
    for n in notes:
        by_row.setdefault(n.row, []).append(n)
    for x in msgs:
        if x.flags & abi.EVF_NEXT_EVENT:
            nexts.setdefault(x.row, []).append(next_view(x, dt))
        elif x.type in CHECKED:
            sent.setdefault((x.row % G, x.from_slot), []).append(msg_view(x, G, di, dt))
    bad = []
    for g, (c, S, s) in enumerate(zip(cases, want, rows)):
        ns = by_row.get(s.row, [])
        fatal = next((n.c & 0xff for n in ns if n.type == abi.NOTE_STATUS and n.aux & abi.ST_FATAL), 0)
        if S.fatal or fatal:
            got, exp = dict(fatal=fatal, flag=bool(s.flags & 4)), dict(fatal=S.fatal, flag=bool(S.fatal))
        else:
            got, exp = row_view(s, di, dt), model_view(S)
            bits = 0
            for n in ns:
                bits |= n.aux
            got["status"], exp["status"] = bits & STATUS_BITS, S.status
            if records:
                got["msgs"], exp["msgs"] = sent.get((g, c.S.me), []), [x for x in S.msgs if x[0] in CHECKED]
            if pure:
                got["nexts"], exp["nexts"] = nexts.get(s.row, []), [model_next(k, e) for k, e in S.nexts]
        if got != exp:
            diff = {k: (exp[k], got.get(k)) for k in exp if exp[k] != got.get(k)}
            bad.append("case %d %s: %s (rule, got)" % (g, c.desc, diff))
    assert not bad, "M=%d %s %s: %d of %d cases differ from the rule, e.g.\n  %s" % (
        m, setting, b.name, len(bad), len(cases), "\n  ".join(bad[:6]))


REACHED = [
    "vote granted: log up to date", "vote declined: already voted", "vote declined: log behind",
    "vote declined: lower term", "vote declined: leader", "vote declined: candidate", "vote ignored: not a voter",
    "pre_vote granted: machine version equal", "pre_vote granted: machine version in range",
    "pre_vote declined: protocol version", "pre_vote declined: machine version above ours",
    "pre_vote declined: machine version below effective", "pre_vote declined: follower stays silent",
    "pre_vote declined: log behind", "pre_vote declined: lower term", "pre_vote ignored: not a voter",
    "election: pre_vote", "election: candidate", "election timeout ignored: not a voter",
    "pre_vote counted", "pre_vote wins", "candidate wins", "pre_vote not counted: token",
    "pre_vote not counted: not a voter",
    "back-off: last index not found", "back-off: same term", "back-off: below match_index",
    "back-off: other term above match_index", "back-off: unknown slot", "snapshot sent",
    "AppendEntries from the snapshot", "AppendEntries from the log",
    "step down: reply", "step down: AppendEntries", "step down: request_vote", "step down: pre_vote",
    "step down: heartbeat", "higher-term request from an unknown slot ignored", "enforce leadership",
    "fatal: AppendEntries in the same term", "fatal: heartbeat in the same term",
    "redispatch from leader", "redispatch from candidate", "redispatch from pre_vote",
    "redispatch from await_condition",
    "AppendEntries prev ok", "AppendEntries prev missing", "AppendEntries prev term_mismatch",
    "AppendEntries at a lower term",
    "condition timeout: reply resent", "condition timeout: nothing to resend", "condition met: ok",
    "condition met: term_mismatch", "condition not met",
]


def _coverage(m, want):
    """every arm of the restated clauses is reached (the oracle matched the rule on each)"""
    seen = set()
    for S in want:
        seen |= S.tags
    need = set(REACHED)
    if m == 1:                                          # one member: no other voter, no other peer to back off
        need -= {"vote declined: already voted", "pre_vote counted", "back-off: same term",
                 "back-off: below match_index", "back-off: other term above match_index", "back-off: last index not found",
                 "snapshot sent", "AppendEntries from the snapshot", "AppendEntries from the log",
                 "step down: reply", "step down: request_vote", "step down: pre_vote", "redispatch from leader",
                 "pre_vote not counted: token", "pre_vote not counted: not a voter"}
        need |= {"pre_vote wins", "candidate wins"}
    assert need <= seen, "M=%d: the table does not reach %s" % (m, sorted(need - seen))


def narrow_pass(backend, m, kw, wide):
    """does this backend step M-member rows in the 32-bit pass?  The engine has it for M = 5 (routed and host-routed)
    and M = 3, 7 (routed), the emulation for M = 5; pure mode too, where every event then stalls."""
    if wide != "0":
        return False
    routed = kw.get("route_on_device", False)
    return m == 5 or (backend == "engine" and routed and m in (3, 7))


def run_table(backend, setting, m, monkeypatch):
    kw, wide, shift, _ = SETTINGS[setting]
    pure = kw.get("pure", False)
    records = not kw.get("route_on_device", False) or pure
    monkeypatch.setenv("RA_STEP_WIDE", wide)
    G, cases = table(m)
    di, dt = shift or (0, 0)
    rows, events = [], []
    for g, c in enumerate(cases):
        r = c.S.row(c.S.me * G + g)
        x = to_event(r.row, c.ev)
        if shift:
            shift_state(r, di, dt, m)
            shift_event(x, di, dt)
        rows.append(r)
        events.append(x)
    want = expect(cases, pure)
    o = Oracle(G, m, **kw)
    bs = [o] if backend == "oracle" else [o, make_backend(backend, G, m, **kw)]
    outs = []
    for b in bs:
        b.load_rows(rows)
        b.load_query_state([])
        outs.append(b.step([clone(e) for e in events]))
    b = bs[-1]
    _check_rule(b, m, setting, G, cases, want, outs[-1], records, pure, di, dt)
    cnt = b.counters()
    total = sum((S.cnt for S in want), Counter())
    assert {k: cnt[k] for k in COUNTERS} == {k: total[k] for k in COUNTERS}, "M=%d %s %s: counters" % (
        m, setting, b.name)
    if backend == "oracle":
        if not shift and not pure:                      # (pure mode chases nothing: no redispatch, no won election)
            _coverage(m, want)
        return
    compare(observe(o, m, outs[0]), observe(b, m, outs[1]), "M=%d %s %s" % (m, setting, backend), events, o)
    narrow = narrow_pass(backend, m, kw, wide)
    if shift and narrow:                                # every row is wide: the general kernel takes it, uncounted
        exp = Counter()
    else:
        exp = Counter(k for k in (hot_event(c.S, c.ev, narrow, pure) for c in cases) if k is not None)
    hist = b.stall_histogram()
    assert hist == dict(exp), "M=%d %s: general-kernel events by (role, type): expected %s, got %s" % (
        m, setting, sorted(exp.items()), sorted(hist.items()))


@pytest.mark.parametrize("m", MEMBERS)
@pytest.mark.parametrize("setting", list(SETTINGS))
@pytest.mark.parametrize("backend", ["oracle", "emu"])
def test_election_table(backend, setting, m, monkeypatch):
    run_table(backend, setting, m, monkeypatch)


@pytest.mark.gpu
@pytest.mark.parametrize("m", MEMBERS)
@pytest.mark.parametrize("setting", list(SETTINGS))
def test_election_table_engine(setting, m, monkeypatch):
    run_table("engine", setting, m, monkeypatch)


# ---- senders a row cannot hold ----------------------------------------------------------------------------------------
def run_rejected(backend, monkeypatch):
    """A batch with an event from a sender slot in 15..254 is RA_E_INVAL and changes no row; the same batch without
    that event steps normally (and equals the oracle)."""
    monkeypatch.setenv("RA_STEP_WIDE", "0")
    m, G = 5, 16
    rng = random.Random(77)
    o = Oracle(G, m)
    bs = [o] if backend == "oracle" else [o, make_backend(backend, G, m)]
    cases = [table(m)[1][k] for k in range(G)]
    rows = [c.S.row(c.S.me * G + g) for g, c in enumerate(cases)]
    good = [to_event(r.row, c.ev) for r, c in zip(rows, cases)]
    for b in bs:
        b.load_rows(rows)
        b.load_query_state([])
    for slot in (15, 16, 17, 31, 200, 254):
        k = rng.randrange(G)
        bad = [clone(e) for e in good]
        bad[k] = abi.ev_request_vote(good[k].row, slot, T, LAST, LT)
        for b in bs:
            before = b.rows_bytes()
            with pytest.raises(abi.RaError) as ei:
                b.step([clone(e) for e in bad])
            assert ei.value.status == abi.RA_E_INVAL, (b.name, slot)
            assert b.rows_bytes() == before, (b.name, slot)
    evs = [e for i, e in enumerate(good) if i % 3]
    outs = [b.step([clone(e) for e in evs]) for b in bs]
    assert o.counters()["events"] >= len(evs)
    if backend != "oracle":
        compare(observe(o, m, outs[0]), observe(bs[1], m, outs[1]), "after the rejected batches", evs, o)


@pytest.mark.parametrize("backend", ["oracle", "emu"])
def test_sender_slot_rejected(backend, monkeypatch):
    run_rejected(backend, monkeypatch)


@pytest.mark.gpu
def test_sender_slot_rejected_engine(monkeypatch):
    run_rejected("engine", monkeypatch)
