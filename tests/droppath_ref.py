"""Python restatement of ivb_droppath_plan: the liveness rules of a DropPath plan over M rows (include/ivb200.h)."""
import numpy as np


def plan(rowscale):
    """rowscale: the M per-row factors of one branch -> (tile order [nm], live tiles, k-block list [live k-blocks]).
    A row is live when its factor is not 0; a 128-row tile or 64-row k-block when one of its rows is."""
    live_row = np.asarray(rowscale, dtype=np.float32) != 0
    M = live_row.size
    nm, nk = (M + 127) // 128, (M + 63) // 64
    tile_live = [bool(live_row[128 * t:128 * t + 128].any()) for t in range(nm)]
    kb_live = [bool(live_row[64 * k:64 * k + 64].any()) for k in range(nk)]
    order = [t for t in range(nm) if tile_live[t]] + [t for t in range(nm) if not tile_live[t]]
    return order, sum(tile_live), [k for k in range(nk) if kb_live[k]]


def clip_rows(keep, n, scale=1.25):
    """Per-row factors of a per-clip draw keep [B] (bool) over clips of n rows: the EPI_RESID rowscale."""
    return np.repeat(np.where(np.asarray(keep), np.float32(scale), np.float32(0)), n)


def flat(order, live, klist, M):
    """The plan as ivb_droppath_plan writes it: order, live count, k-block list padded to nk slots, count.  The slots
    past the count are not written by the kernel: -1 here, and the comparison skips them."""
    nk = (M + 63) // 64
    return np.array(order + [live] + klist + [-1] * (nk - len(klist)) + [len(klist)], dtype=np.int32)
