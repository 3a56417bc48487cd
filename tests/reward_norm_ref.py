"""numpy float64 reference of fxenv_return_moments (include/fxenv.h): the discounted-return scan of the reward
normalizer, vectorised over the envs of a slice (each env's recursion is elementwise, one rounding per operation)."""
import numpy as np


def return_scan(reward, done, prev_done, ret, seen, begun, gamma, shift):
    """reward float32 [H, W], done uint8 [H, W], prev_done [W], ret float64 [W], seen [W], begun [W] (the slice's
    envs) -> (ret float64 [W], seen int64 [W], out float64 [3] = (sum (R - shift), sum (R - shift)^2, count))"""
    reward = np.asarray(reward, np.float32)
    done = np.asarray(done)
    H, W = reward.shape
    reset = np.empty((H, W), bool)
    reset[0] = np.asarray(prev_done) != 0
    reset[1:] = done[:-1] != 0
    begun = np.asarray(begun, np.int64)
    keep = begun - reset.sum(0) == np.asarray(seen, np.int64)
    R = np.where(keep, np.asarray(ret, np.float64), 0.0)
    g, sh = np.float64(gamma), np.float64(shift)
    s1 = s2 = 0.0
    n = 0
    for t in range(H):
        v = ~reset[t]
        R = np.where(v, R * g + reward[t].astype(np.float64), R)
        d = (R - sh)[v]
        s1 += float(d.sum())
        s2 += float((d * d).sum())
        n += int(v.sum())
        R = np.where(done[t] != 0, 0.0, R)
    return R, begun.copy(), np.array([s1, s2, float(n)])
