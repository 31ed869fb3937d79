"""Seed joins restated over the literal model's name-keyed stores (oracle/core_model.py). TEST INFRASTRUCTURE ONLY: a
second statement of DESIGN.md 2.7, independent of the C oracle's (tests/join_oracle.c), which tests/test_join_model.py
holds the two against. The receive rules and the piggyback queue are tests/push_pull_model.py's."""
from typing import Dict

from oracle.core_model import ALIVE, DEAD, SUSPECT, Msg, Store, members, next_incarnation_prime
from push_pull_model import enqueue, receive


def join(stores: Dict[str, Store], up: Dict[str, bool], pairs, view_cap: int, pb_cap: int, retransmit: int,
         fresh=False, strict=False, lg_delta=None) -> dict:
    """Seed joins between steps (memberlist's Join(joinHosts); DESIGN.md 2.7): pairs = [(joiner, seed)] by name. With
    `fresh` every listed joiner that is up first forgets its members and its queue. Then a snapshot as push_pull takes
    it, and every pair whose two ends are up is an exchange: the joiner receives the seed's state and the seed the
    joiner's. A store processes its distinct senders in ascending name, each message as push_pull processes it. Returns
    the totals {exchanges, inserted, full, applied, refutes, dropped}."""
    if fresh:
        for j, _ in pairs:
            if up[j]:
                stores[j].members.clear()
                stores[j].timers.clear()
                stores[j].conf = {}
                stores[j].queue = []
    snap = {k: ([(m.name, m.alive, m.incarnation) for m in members(s)], s.incarnation) for k, s in stores.items()}
    senders = {}
    tot = dict(exchanges=0, inserted=0, full=0, applied=0, refutes=0, dropped=0)
    for j, s in pairs:
        if up[j] and up[s]:
            tot["exchanges"] += 1
            senders.setdefault(j, set()).add(s)
            senders.setdefault(s, set()).add(j)
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
