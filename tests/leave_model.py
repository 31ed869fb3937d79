"""Graceful leaves restated over the literal model's name-keyed stores (oracle/core_model.py). TEST INFRASTRUCTURE ONLY: a
second statement of DESIGN.md 2.8, independent of the C oracle's (tests/leave_oracle.c), which tests/test_leave_model.py
holds the two against. The receive rules and the piggyback queue are tests/push_pull_model.py's."""
from typing import Dict

from oracle.core_model import ALIVE, SUSPECT, Msg, Store
from push_pull_model import enqueue, receive


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
