"""Push-pull anti-entropy, seed joins and graceful leaves restated over the literal model's name-keyed stores
(oracle/core_model.py). TEST INFRASTRUCTURE ONLY: a second statement of DESIGN.md 2.6-2.8, independent of the C oracle's
(tests/between_steps_oracle.c), which tests/test_push_pull_model.py, test_join_model.py and test_leave_model.py hold the
two against; the helpers at the end carry an oracle's state into stores and back for them. A store's piggyback buffer
is kept on it as `queue`."""
from typing import Callable, Dict, Optional

from dataclasses import replace

import numpy as np

from oracle.core_model import (ALIVE, DEAD, SUSPECT, Member, Msg, Store, alive_node, dead_node, members,
                               next_incarnation_prime, suspect_node)
from oracle.oracle import Oracle
from swim_b200 import _abi as A
from swim_b200.sim import crash_events, default_config, generate_topology

NM = A.NO_MEMBER
KIND = {A.MSG_ALIVE: "Alive", A.MSG_SUSPECT: "Suspect", A.MSG_DEAD: "Dead"}


def enqueue(s: Store, msg: Msg, cap: int, retransmit: int) -> int:
    """[Q5] the piggyback buffer `Broadcast m` should have fed (Core.hs:131,136-138): newest first, a newer message about
    the same member replaces the older one, the oldest falls off a full buffer. s.queue holds (msg, transmissions left).
    Returns 1 when a message fell off."""
    q = [(m, t) for m, t in getattr(s, "queue", []) if m.node != msg.node]
    dropped = len(q) == cap
    s.queue = [(msg, retransmit)] + q[: cap - 1]
    return int(dropped)


def confirm(s: Store, name: str, lg_delta) -> None:
    """[Lifeguard] a further Suspect about a suspected member: the c-th confirmation (c <= 3) takes lg_delta[c] off the
    countdown, never below 1. s.conf holds the confirmations seen per member."""
    c = s.conf.get(name, 0)
    if c < 3:
        s.conf[name] = c + 1
        s.timers[name] = max(s.timers[name] - lg_delta[c + 1], 1)


def receive(s: Store, msg: Msg, strict=False, lg_delta=None) -> Optional[Msg]:
    """One Suspect / Dead / Alive about another member, as received from the network. The reference's guards
    (core_model) unless `strict`: the SWIM paper's overrides (section 4.2, SWIM_F_STRICT_OVERRIDE in include/swim.h).
    lg_delta (suspicion_max > 0): a Suspect that is `Nothing` about a member already Suspect counts as a confirmation."""
    if not hasattr(s, "conf"):
        s.conf = {}
    m = s.members.get(msg.node)
    i = msg.incarnation
    if m is not None and msg.kind == "Suspect" and lg_delta and m.alive == SUSPECT:
        if (i == m.incarnation) if strict else (i >= m.incarnation):
            confirm(s, msg.node, lg_delta)
            return None
    if m is None or not strict:
        out = {"Alive": alive_node, "Suspect": suspect_node, "Dead": dead_node}[msg.kind](s, msg)
    elif msg.kind == "Suspect":
        if m.alive == DEAD or (i < m.incarnation if m.alive == ALIVE else i <= m.incarnation):
            return None
        s.members[msg.node] = replace(m, incarnation=i, alive=SUSPECT, last_change=s.now)
        s.timers[msg.node] = s.S
        out = msg
    elif msg.kind == "Dead":
        if m.alive == DEAD:
            return None
        s.members[msg.node] = replace(m, incarnation=max(i, m.incarnation), alive=DEAD, last_change=s.now)
        s.timers.pop(msg.node, None)
        out = msg
    else:
        if i <= m.incarnation:
            return None
        s.members[msg.node] = replace(m, incarnation=i, alive=ALIVE, last_change=s.now)
        s.timers.pop(msg.node, None)
        out = msg
    if out is not None:
        s.conf.pop(msg.node, None)
    return out


def snapshot(stores: Dict[str, Store]) -> dict:
    """Every store's state as an exchange sends it: ([(name, alive, incarnation)] in key order, own incarnation)."""
    return {k: ([(m.name, m.alive, m.incarnation) for m in members(s)], s.incarnation) for k, s in stores.items()}


def exchange(stores: Dict[str, Store], snap: dict, senders: Dict[str, set], view_cap: int, pb_cap: int, retransmit: int,
             tot: dict, strict=False, lg_delta=None) -> dict:
    """Every receiver j of `senders` processes the snapshot states of its senders in ascending name: Alive about the
    sender, then every member as Alive / Suspect / Dead(deadFrom = sender), each message as `process` would (its own
    entry is virtual: Alive at storeIncarnation), with a `Just` enqueued; an insert into a store already holding
    view_cap members is dropped. `strict` and `lg_delta` select the protocol variants (`receive`). Adds inserted, full,
    applied, refutes and dropped to `tot`, and returns it."""
    kinds = {ALIVE: "Alive", SUSPECT: "Suspect", DEAD: "Dead"}
    for j in sorted(senders):
        s = stores[j]
        for snd in sorted(senders[j]):
            ms, inc = snap[snd]
            msgs = [Msg("Alive", node=snd, incarnation=inc)]
            msgs += [Msg(kinds[lv], node=name, incarnation=i, dead_from=snd if lv == DEAD else "") for name, lv, i in ms]
            for msg in msgs:
                if msg.node == j:                      # own entry: (Alive, storeIncarnation)
                    if msg.kind == "Alive" or (msg.incarnation < s.incarnation and not (strict and msg.kind == "Dead")):
                        continue
                    out = Msg("Alive", node=j, incarnation=next_incarnation_prime(s, msg.incarnation))
                    tot["refutes"] += 1
                else:
                    if msg.kind == "Alive" and msg.node not in s.members:   # addNewMember, Core.hs:206-216
                        if len(s.members) == view_cap:
                            tot["full"] += 1
                            continue
                        tot["inserted"] += 1
                    out = receive(s, msg, strict, lg_delta)
                if out is not None:
                    tot["applied"] += 1
                    tot["dropped"] += enqueue(s, out, pb_cap, retransmit)
    return tot


def _totals(exchanges):
    return dict(exchanges=exchanges, inserted=0, full=0, applied=0, refutes=0, dropped=0)


def push_pull(stores: Dict[str, Store], up: Dict[str, bool], draw: Callable[[str], int], view_cap: int,
              pb_cap: int, retransmit: int, strict=False, lg_delta=None) -> dict:
    """Push-pull anti-entropy between steps (memberlist's periodic full-state exchange; DESIGN.md 2.6). No reference
    counterpart: Config.joinHosts (Types.hs:47) is parsed and never used, so nothing feeds aliveNode's insertion
    (Core.hs:206-216) with members a store does not know. Every up store with Alive members picks the
    (draw(name) * L >> 32)-th of them in key order; when that partner is up the two exchange their states, both taken
    from a snapshot made first (`exchange`). Returns the totals {exchanges, inserted, full, applied, refutes, dropped}."""
    snap = snapshot(stores)
    partner = {}
    for k in sorted(stores):
        if not up[k]:
            continue
        alive = [name for name, lv, _ in snap[k][0] if lv == ALIVE]
        if alive:
            p = alive[(draw(k) * len(alive)) >> 32]
            if up[p]:
                partner[k] = p
    senders = {}
    for k, p in partner.items():
        senders.setdefault(k, set()).add(p)
        senders.setdefault(p, set()).add(k)
    return exchange(stores, snap, senders, view_cap, pb_cap, retransmit, _totals(len(partner)), strict, lg_delta)


def join(stores: Dict[str, Store], up: Dict[str, bool], pairs, view_cap: int, pb_cap: int, retransmit: int,
         fresh=False, strict=False, lg_delta=None) -> dict:
    """Seed joins between steps (memberlist's Join(joinHosts); DESIGN.md 2.7): pairs = [(joiner, seed)] by name. With
    `fresh` every listed joiner that is up first forgets its members and its queue. Then a snapshot as push_pull takes
    it, and every pair whose two ends are up is an exchange: the joiner receives the seed's state and the seed the
    joiner's (`exchange`: each distinct sender once). Returns the totals {exchanges, inserted, full, applied, refutes,
    dropped}."""
    if fresh:
        for j, _ in pairs:
            if up[j]:
                stores[j].members.clear()
                stores[j].timers.clear()
                stores[j].conf = {}
                stores[j].queue = []
    snap = snapshot(stores)
    senders = {}
    exchanges = 0
    for j, s in pairs:
        if up[j] and up[s]:
            exchanges += 1
            senders.setdefault(j, set()).add(s)
            senders.setdefault(s, set()).add(j)
    return exchange(stores, snap, senders, view_cap, pb_cap, retransmit, _totals(exchanges), strict, lg_delta)


def leave(stores: Dict[str, Store], up: Dict[str, bool], names, pb_cap: int, retransmit: int, strict=False,
          lg_delta=None) -> dict:
    """Graceful leaves between steps (memberlist's Leave; DESIGN.md 2.8): the leavers are the listed stores that are up,
    each once. All of them go down first (`up` is updated in place). Then every up store, for each leaver that holds it
    Alive or Suspect, in ascending leaver name, processes Dead(leaver's incarnation, leaver, deadFrom = leaver) as a
    received datagram: a message about a member it does not know is `Nothing`, a `Just` is enqueued. Returns
    {left: the leavers in ascending name, delivered, applied, dropped}."""
    left = sorted({k for k in names if up[k]})
    for k in left:
        up[k] = False
    tot = dict(left=left, delivered=0, applied=0, dropped=0)
    for j in sorted(stores):
        if not up[j]:
            continue
        s = stores[j]
        for L in left:
            held = stores[L].members.get(j)
            if held is None or held.alive not in (ALIVE, SUSPECT):
                continue
            tot["delivered"] += 1
            if L not in s.members:
                continue
            out = receive(s, Msg("Dead", node=L, incarnation=stores[L].incarnation, dead_from=L), strict, lg_delta)
            if out is not None:
                tot["applied"] += 1
                tot["dropped"] += enqueue(s, out, pb_cap, retransmit)
    return tot


# ------------------------------------------------------------------ an oracle's state as stores, and back
def name(i):
    return f"{i:05d}"  # key order == id order


def lifeguard_deltas(cfg):
    """What the c-th confirmation takes off a countdown: timeout(c) = max - (max - min) log(c + 1) / log 4, c = 0..3, in
    256ths rounded (the oracle's table)."""
    if not cfg.suspicion_max:
        return None
    frac = (0, 128, 203, 256)
    T = [cfg.suspicion_max - ((cfg.suspicion_max - cfg.suspicion_rounds) * f + 128) // 256 for f in frac]
    return [0] + [T[c - 1] - T[c] for c in range(1, 4)]


def to_model(orc, cfg):
    n, cap = cfg.n_nodes, cfg.view_cap
    lg = cfg.suspicion_max != 0
    nb, st, inc, last = (orc.get_array(a).reshape(n, cap) for a in (A.ARR_NBR, A.ARR_VST, A.ARR_VINC, A.ARR_VLAST))
    pb, cnt = orc.get_array(A.ARR_PB).reshape(n, cfg.pb_cap), orc.get_array(A.ARR_PB_CNT)
    stores = {}
    for i in range(n):
        s = Store(Member(name(i)), cfg.suspicion_max or cfg.suspicion_rounds)
        s.conf = {}
        s.incarnation = int(orc.get_array(A.ARR_SELF_INC)[i])
        s.now = orc.round
        for x in range(cap):
            if st[i, x] & 3 == A.VACANT:
                continue
            m = name(int(nb[i, x]))
            s.members[m] = Member(m, "", 0, 0, int(st[i, x] & 3), int(inc[i, x]), int(last[i, x]))
            if st[i, x] & 3 == A.SUSPECT:
                s.timers[m] = (int(st[i, x]) >> 2) & (15 if lg else 63)
                if lg and st[i, x] >> 6:
                    s.conf[m] = int(st[i, x]) >> 6
        s.queue = [(Msg(KIND[int(r["kind"])], node=name(int(r["member"])), incarnation=int(r["incarnation"]),
                          dead_from=name(int(r["from"])) if r["kind"] == A.MSG_DEAD else ""), int(r["ttl"]))
                   for r in pb[i, : cnt[i]]]
        stores[name(i)] = s
    return stores


def model_arrays(stores, cfg):
    n, cap = cfg.n_nodes, cfg.view_cap
    nb = np.full((n, cap), NM, np.uint32)
    st = np.full((n, cap), A.VACANT, np.uint8)
    inc = np.zeros((n, cap), np.uint32)
    last = np.zeros((n, cap), np.uint32)
    pb = []
    for i in range(n):
        s = stores[name(i)]
        for x, m in enumerate(members(s)):
            nb[i, x], inc[i, x], last[i, x] = int(m.name), m.incarnation, m.last_change
            if m.alive == A.SUSPECT:
                st[i, x] = m.alive | (s.timers.get(m.name, 0) << 2) | (s.conf.get(m.name, 0) << 6)
            else:
                st[i, x] = m.alive
        pb.append([(int(m.node), {"Alive": A.MSG_ALIVE, "Suspect": A.MSG_SUSPECT, "Dead": A.MSG_DEAD}[m.kind],
                    m.incarnation, int(m.dead_from) if m.kind == "Dead" else 0, t) for m, t in s.queue])
    self_inc = np.array([stores[name(i)].incarnation for i in range(n)], np.uint32)
    return nb, st, inc, last, self_inc, pb


def oracle_pb(orc, cfg):
    pb, cnt = orc.get_array(A.ARR_PB).reshape(cfg.n_nodes, cfg.pb_cap), orc.get_array(A.ARR_PB_CNT)
    return [[(int(r["member"]), int(r["kind"]), int(r["incarnation"]), int(r["from"]), int(r["ttl"])) for r in pb[i, : cnt[i]]]
            for i in range(cfg.n_nodes)]


def variant(cfg):
    """The protocol variant of a config, as push_pull, join and leave take it."""
    return dict(strict=bool(cfg.flags & A.F_STRICT_OVERRIDE), lg_delta=lifeguard_deltas(cfg))


def up_of(orc):
    return {name(i): bool(a) for i, a in enumerate(orc.get_array(A.ARR_ALIVE))}


def assert_same_state(orc, stores, cfg):
    """Every view entry, incarnation and piggyback buffer of the oracle equals the stores'."""
    nb, st, inc, last, self_inc, pb = model_arrays(stores, cfg)
    n, cap = cfg.n_nodes, cfg.view_cap
    assert np.array_equal(orc.get_array(A.ARR_NBR).reshape(n, cap), nb)
    assert np.array_equal(orc.get_array(A.ARR_VST).reshape(n, cap), st)
    assert np.array_equal(orc.get_array(A.ARR_VINC).reshape(n, cap), inc)
    assert np.array_equal(orc.get_array(A.ARR_VLAST).reshape(n, cap), last)
    assert np.array_equal(orc.get_array(A.ARR_SELF_INC), self_inc)
    assert oracle_pb(orc, cfg) == pb


def setup(n, kind, deg, seed=1, rounds=0, crashes=(), cap=32, **kw):
    cfg = default_config(n_nodes=n, view_cap=cap, seed=seed, suspicion_rounds=4, **kw)
    orc = Oracle(cfg)
    orc.set_view(generate_topology(kind, n, cap, deg, seed=seed))
    if crashes:
        orc.inject(crash_events(1, list(crashes)))
    if rounds:
        orc.step(rounds)
    return orc, cfg
