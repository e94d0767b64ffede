"""CPU: the generators of the post-processing conformance suite land where tests/test_gpu_post_conformance.py says they do, and the
decode bounds of tests/post_conformance_cases.py have teeth -- a float32 emulation of the kernels (also with its sums in reverse order)
passes them, and each deliberately wrong decode fails them."""
import time

import numpy as np
import pytest

import post_conformance_cases as pc
import synth
from oracle import post, track


@pytest.mark.parametrize("hits", [2047, 2048, 2049, 5000, 8400])
def test_v8_selection_generator_hits_exact_counts(hits):
    raw = pc.v8_selection_raw(hits, hits)
    boxes, cls, confs = post.yolo_process_output(raw, "v8", 0.4)
    assert len(confs) == hits


def test_v5_selection_generator_hits_exact_counts():
    assert len(post.yolo_process_output(pc.v5_selection_raw(1, 2600), "v5", 0.4)[2]) == 2600
    assert len(post.yolo_process_output(pc.v5_selection_raw(2, 1500), "v5", 0.4)[2]) == 1500
    assert len(post.yolo_process_output(pc.v5_selection_raw(3, 3000, A=102000, in_hw=(1280, 1280)), "v5", 0.4)[2]) == 3000


def test_tie_generator_counts_and_strict_threshold():
    bs = float(np.float32(0.45))
    raw, n = pc.v8_tie_raw(3, bs)
    boxes, cls, confs = post.yolo_process_output(raw, "v8", bs)
    assert len(confs) == n and sum(c == 1.0 for c in confs) == 600
    assert bs not in confs and float(np.nextafter(np.float32(bs), np.float32(1))) in confs


def test_crowd_sequence_reaches_the_association_routes():
    """the sequence of the GPU tracker test drives the pool and the unconfirmed list past the 120 rows of shared memory and the removed
    list past its 4096-entry trim"""
    seq = pc.crowd_sequence(7, objects=300, frames=64, clutter=150)
    _, pmax, umax, nrem = pc.run_oracle(track.Tracker, seq)
    assert pmax > 120 and umax > 120 and nrem > 4096, (pmax, umax, nrem)


def test_crafted_head_logits_are_float16_exact_and_reach_the_edges():
    """the identity-conv plan of the GPU test feeds these through fp16: they must survive the round trip, and they must contain the
    saturating / underflowing class logits and the DFL patterns"""
    g = pc.crafted_head(40, "v8", 8, 12, 80, 16)
    assert np.array_equal(g, g.astype(np.float16).astype(np.float32))
    cls = g[..., 64:80]
    assert {30.0, -30.0, 88.5, -88.5, -89.0, 104.0}.issubset(set(cls.ravel().tolist()))
    dfl = g[..., :64].reshape(-1, 16)
    assert (dfl.max(1) == dfl.min(1)).any() and (dfl.argmax(1) == 0).any() and (dfl.argmax(1) == 15).any()


LEVEL_KINDS = [("v8", 16, (256, 384), (8, 16, 32)), ("v6", 0, (256, 384), (8, 16, 32)), ("v6", 16, (256, 384), (8, 16, 32)),
               ("v5", 16, (256, 384), (8, 16, 32)), ("v5", 16, (256, 256), (8, 16, 32, 64))]


@pytest.mark.parametrize("kind,reg_max,in_hw,strides", LEVEL_KINDS)
def test_decode_bounds_pass_float32_emulation(kind, reg_max, in_hw, strides):
    lv = pc.random_levels(11, kind, in_hw=in_hw, reg_max=reg_max, strides=strides)
    an = np.concatenate([post.V5_ANCHORS, post.V5_ANCHORS[-1:] * 2])[:len(strides)]
    ref, bnd = pc.decode_reference(kind, lv, 80, reg_max, an)
    for rev in (False, True):
        ex, _ = pc.decode_excess(pc.emulate_decode(kind, lv, 80, reg_max, an, reverse_sums=rev), ref, bnd)
        assert ex <= 1.0, (kind, reg_max, rev, ex)


MUTATIONS = {"v8": ["anchor_offset_0", "stride_off_by_one_level", "xy_swapped", "dfl_15_bins"],
             "v6": ["anchor_offset_0", "stride_off_by_one_level", "xy_swapped"],
             "v5": ["stride_off_by_one_level", "xy_swapped", "anchor_wh_swapped"]}


@pytest.mark.parametrize("kind,reg_max,in_hw,strides", LEVEL_KINDS)
def test_decode_bounds_catch_wrong_decodes(kind, reg_max, in_hw, strides):
    lv = pc.random_levels(12, kind, in_hw=in_hw, reg_max=reg_max, strides=strides)
    an = np.concatenate([post.V5_ANCHORS, post.V5_ANCHORS[-1:] * 2])[:len(strides)]
    ref, bnd = pc.decode_reference(kind, lv, 80, reg_max, an)
    muts = MUTATIONS[kind] + (["dfl_15_bins"] if kind == "v6" and reg_max == 16 else [])
    if in_hw[0] == in_hw[1]:
        muts = [m for m in muts if m != "xy_swapped"]               # only a non-square grid can tell x from y by shape
    for m in muts:
        ex, _ = pc.decode_excess(pc.emulate_decode(kind, lv, 80, reg_max, an, mutation=m), ref, bnd)
        assert ex > 1.0, (kind, reg_max, m, ex)


def test_oracle_soft_nms_time_at_full_anchor_counts():
    """The GPU test calls the O(n^2) numpy soft_nms on every candidate of 8400- and 25 200-anchor heads; keep those calls short.
    Measured on one x86 core with numpy: 0.4-0.7 s at 8400 candidates and 3.8-4.6 s at 25 200.  The GPU test therefore runs all 8400 candidates
    once and keeps the 25 200- and 102 000-anchor heads at a few thousand candidates."""
    for n, limit in ((8400, 20.0), (25200, 60.0)):
        b, c = synth.nms_case(5, n)
        t0 = time.perf_counter()
        post.soft_nms(b, c, 0.45)
        dt = time.perf_counter() - t0
        print(f"[time] oracle soft_nms on {n} candidates: {dt:.2f} s")
        assert dt < limit
