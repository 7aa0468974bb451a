"""Binomial checkpointing schedules (Griewank & Walther, "Algorithm 799: revolve", ACM TOMS 26(1), 2000).

Reversing `l` time steps of a forward propagation needs, at adjoint step `i` (from l-1 down to 0), the forward state
`i`: the state the forward step `i` starts from. With `s` checkpoints (one of them holding the initial state 0) the
least number of forward steps that makes every state available in reverse order is

    r * l - beta(s + 1, r - 1),    beta(s, r) = C(s + r, s),    r = the least integer with beta(s, r) >= l,

and `schedule` returns a list of actions that reaches it. With s >= l it checkpoints every state and recomputes nothing
(l - 1 forward steps).

The actions, in step indices (state t = after t forward steps):

    ('advance', t0, t1)   run forward steps t0 .. t1-1 (the current state is t0)
    ('takeshot', k, t)    store the current state t in checkpoint k
    ('restore', k)        make the state stored in checkpoint k current
    ('reverse', t)        one adjoint step; it reads forward state t, which is current
"""
from math import comb

__all__ = ['beta', 'repetitions', 'optimal_forward_steps', 'schedule', 'default_n_checkpoints']


def beta(s, r):
    """Steps that s checkpoints reverse with at most r forward recomputations of each step: C(s + r, s)."""
    return comb(s + r, s) if r >= 0 else 0


def repetitions(l, s):
    """The least r with beta(s, r) >= l."""
    r = 0
    while beta(s, r) < l:
        r += 1
    return r


def optimal_forward_steps(l, s):
    """The least number of forward steps that reverses l steps with s checkpoints."""
    if l <= 1:
        return 0
    r = repetitions(l, s)
    return r * l - beta(s + 1, r - 1)


def _split(l, s):
    """Where the first checkpoint goes when l >= 2 steps are reversed with s >= 2 checkpoints. The right part
    (l - m steps, s - 1 checkpoints) must cost r repetitions at most and the left one (m steps, s checkpoints) r - 1:
    m in [beta(s, r-2), beta(s, r-1)] and l - m in [beta(s-1, r-1), beta(s-1, r)]; then the total is
    m + (r-1) m - beta(s+1, r-2) + r (l-m) - beta(s, r-1) = r l - beta(s+1, r-1), the optimum."""
    r = repetitions(l, s)
    return max(1, beta(s, r - 2), l - beta(s - 1, r))


def schedule(l, s):
    """The actions that reverse `l` steps with `s` >= 1 checkpoints in the optimal number of forward steps."""
    l, s = int(l), int(s)
    if s < 1:
        raise ValueError(f"at least one checkpoint is needed, got {s}")
    if l < 1:
        return []
    out = []
    if l > 1:
        out.append(('takeshot', 0, 0))
    # work items: ('rev', a, n, k, c) reverses steps a .. a+n-1 with state a current and stored in checkpoint k,
    # and c checkpoints (k .. k+c-1) for the job; ('restore', k). An explicit stack: the depth reaches l when s >= l.
    work = [('rev', 0, l, 0, s)]
    while work:
        item = work.pop()
        if item[0] == 'restore':
            out.append(item)
            continue
        _, a, n, k, c = item
        if n == 1:
            out.append(('reverse', a))
        elif c == 1:
            # one checkpoint: walk from state a to each state in turn, last first
            for j in range(n - 1, -1, -1):
                if j < n - 1:
                    out.append(('restore', k))
                if j > 0:
                    out.append(('advance', a, a + j))
                out.append(('reverse', a + j))
        else:
            m = _split(n, c)
            out.append(('advance', a, a + m))
            if n - m > 1:
                out.append(('takeshot', k + 1, a + m))
            # popped in turn: the right part, back to state a, the left part
            work.append(('rev', a, m, k, c))
            work.append(('restore', k))
            work.append(('rev', a + m, n - m, k + 1, c - 1))
    return out


def default_n_checkpoints(l, free_bytes, slot_bytes):
    """Checkpoints of two wavefield slots each that fit in 90 % of `free_bytes`, at most one per step."""
    return int(min(int(l), (0.9 * free_bytes) // (2 * slot_bytes)))
