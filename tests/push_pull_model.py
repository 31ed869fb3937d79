"""Push-pull anti-entropy restated over the literal model's name-keyed stores (oracle/core_model.py). TEST
INFRASTRUCTURE ONLY: a second statement of DESIGN.md 2.6, independent of the C oracle's (tests/push_pull_oracle.c), which
tests/test_push_pull_model.py holds the two against. A store's piggyback buffer is kept on it as `queue`."""
from typing import Callable, Dict, Optional

from dataclasses import replace

from oracle.core_model import (ALIVE, DEAD, SUSPECT, Msg, Store, alive_node, dead_node, members,
                               next_incarnation_prime, suspect_node)


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


def push_pull(stores: Dict[str, Store], up: Dict[str, bool], draw: Callable[[str], int], view_cap: int,
              pb_cap: int, retransmit: int, strict=False, lg_delta=None) -> dict:
    """Push-pull anti-entropy between steps (memberlist's periodic full-state exchange; DESIGN.md 2.6). No reference
    counterpart: Config.joinHosts (Types.hs:47) is parsed and never used, so nothing feeds aliveNode's insertion
    (Core.hs:206-216) with members a store does not know. Every up store with Alive members picks the
    (draw(name) * L >> 32)-th of them in key order; when that partner is up the two exchange their states, both taken
    from a snapshot made first: Alive about itself, then every member as Alive / Suspect / Dead(deadFrom = sender). A
    receiver processes its senders in ascending name, each message as `process` would (its own entry is virtual:
    Alive at storeIncarnation), with a `Just` enqueued; an insert into a store already holding view_cap members is
    dropped. `strict` and `lg_delta` select the protocol variants (`receive`). Returns the totals
    {exchanges, inserted, full, applied, refutes, dropped}."""
    snap = {k: ([(m.name, m.alive, m.incarnation) for m in members(s)], s.incarnation) for k, s in stores.items()}
    partner = {}
    for k in sorted(stores):
        if not up[k]:
            continue
        alive = [name for name, lv, _ in snap[k][0] if lv == ALIVE]
        if alive:
            p = alive[(draw(k) * len(alive)) >> 32]
            if up[p]:
                partner[k] = p
    tot = dict(exchanges=len(partner), inserted=0, full=0, applied=0, refutes=0, dropped=0)
    kinds = {ALIVE: "Alive", SUSPECT: "Suspect", DEAD: "Dead"}
    for j in sorted(stores):
        if not up[j]:
            continue
        s = stores[j]
        senders = {i for i, p in partner.items() if p == j} | ({partner[j]} if j in partner else set())
        for snd in sorted(senders):
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
