"""Float64 restatement of the PPN head op (OP_PPN_HEAD): pose_proposal/model.py:84-93 (sigmoid, split, reshape) and restore_coor
(:111-119) at the engine's input size.  The engine's kernel computes the same formulas in fp32; tests compare against this."""
import numpy as np


def ppn_head_ref(raw, K, n_edge, in_h, in_w):
    """raw [N, C >= 6K + n_edge, gh, gw] (the values the engine's raw buffer holds) -> (boxes [N, 6K, gh, gw], edges [N, n_edge, gh, gw])
    float64.  Box channel t*K + k: t = 0 conf_point, 1 conf_iou, 2 x, 3 y, 4 w, 5 h."""
    raw = np.asarray(raw, np.float64)
    N, _, gh, gw = raw.shape
    with np.errstate(over="ignore"):                 # exp(-v) = inf for v < -709: s = 0, as 1 / (1 + inf)
        s = 1.0 / (1.0 + np.exp(-raw[:, :6 * K + n_edge]))
    box = s[:, :6 * K].reshape(N, 6, K, gh, gw).copy()
    gy, gx = np.meshgrid(np.arange(gh, dtype=np.float64), np.arange(gw, dtype=np.float64), indexing="ij")
    box[:, 2] = (box[:, 2] + gx) * (in_w / gw)
    box[:, 3] = (box[:, 3] + gy) * (in_h / gh)
    box[:, 4] *= in_w
    box[:, 5] *= in_h
    return box.reshape(N, 6 * K, gh, gw), s[:, 6 * K:]
