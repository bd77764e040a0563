"""A numpy restatement of g6d_instances_verify_update (row f21), the slot update of a verifying instance-tracking step."""
import numpy as np


def verify_update(lost, verified, max_misses, live, ids, misses):
    """-> (live, ids, misses, dropped) after the update; the inputs are not modified.  A live slot of a verified row judged
    lost takes a miss and is dropped past max_misses (live 0, id -1, misses 0, its id in dropped); one judged found restarts
    its misses; every other row keeps its state, and dropped is -1 wherever nothing was dropped."""
    live, ids, misses = live.astype(np.int32).copy(), ids.astype(np.int64).copy(), misses.astype(np.int32).copy()
    lost, verified = np.asarray(lost) != 0, np.asarray(verified) != 0
    judged = verified & (live != 0)
    misses[judged & ~lost] = 0
    missed = judged & lost
    misses[missed] += 1
    drop = missed & (misses > max_misses)
    dropped = np.where(drop, ids, -1).astype(np.int64)
    live[drop], ids[drop], misses[drop] = 0, -1, 0
    return live, ids, misses, dropped
