"""Relative errors of a result against its reference, over the whole tensor and over each slice of it.

A relative error over a whole tensor lets an error confined to one slice -- one token row, one output channel of a
weight gradient, one head of a q/k-norm weight -- shrink by the square root of the number of slices: one wrong row
among 834 moves the tensor's error by 1/29 of its own.  slice_errors measures the error of every slice against the
reference's typical slice (its rms over the slices), so such an error reads at full size.  Normalising by the typical
slice rather than by the slice's own reference, as tests/attn_ref.py:tile_errors normalises a band by its whole head,
keeps a slice whose reference happens to be small (a weight-gradient channel whose terms cancel over the tokens) from
reading as a large relative error.
"""
from __future__ import annotations

import torch


def rel(got, ref):
    """||got - ref|| / ||ref|| over the whole tensor, in float64."""
    g, r = got.detach().double(), ref.detach().double().to(got.device)
    return float((g - r).norm() / (r.norm() + 1e-30))


def slice_errors(got, ref, slices):
    """||got_s - ref_s|| / (||ref|| / sqrt(slices)) of each of `slices` equal, contiguous slices of the flattened
    tensors (the rows of a [rows, cols] matrix for slices = rows; the heads of a [H * d] vector for slices = H): each
    slice's error relative to the rms norm of the reference's slices.  float64 [slices]."""
    g = got.detach().double().reshape(slices, -1)
    r = ref.detach().double().to(g.device).reshape(slices, -1)
    return (g - r).norm(dim=1) / (r.norm() / slices ** 0.5 + 1e-30)


def worst_slice(errs):
    """(largest error, its slice index)."""
    i = int(errs.argmax())
    return float(errs[i]), i
