"""Restatement of the actuation delay (rsb_batch_set_actuation_delay, include/rsb.h): at advancing sub-step t since the command history
was last emptied, the actuator applies the command of sub-step max(t - d, 0)."""
import numpy as np


def applied_index(t, d):
    """the sub-step (counted from the last emptying) whose command applies at sub-step t under delay d"""
    return max(t - d, 0)


def applied(commands, delays, empty_before=()):
    """commands [T, ...]: the command of every advancing sub-step of one environment, in order.  delays: the delay in force, an int or
    [T] (it changes only where the history is emptied).  empty_before: the sub-steps just before which the history was emptied (setting
    the delay, a gym reset or a termination); sub-step 0 starts empty.  Returns [T, ...]: the command each sub-step applies."""
    commands = np.asarray(commands)
    T = len(commands)
    d = np.broadcast_to(np.asarray(delays, np.int64), (T,))
    out = np.empty_like(commands)
    start = 0
    for s in range(T):
        if s in empty_before:
            start = s
        out[s] = commands[start + applied_index(s - start, int(d[s]))]
    return out
