"""CPU: the helpers of the rig-size GPU checks (rig_scale_cases.py).  A small YOLOv8-n plan (96 x 128, six images) with the float64
interpreter's outputs, rounded to the plan's dtypes, standing in for the device buffers:
- op_ref on subset(..., [0, 4, 5]) equals op_ref on the whole batch restricted to those images, bit for bit, for every op;
- an error of a few bounds in one element of image 5 of one op's output is reported with that op and image 5;
- two images swapped in one buffer are reported by the per-image digests of stream_read;
and the regrouping schedule of the multi-tracker check has every case it is meant to reach."""
import numpy as np
import pytest

import plan_interp as pi
import rig_scale_cases as rc
import synth
from adas_b200 import plan
from gpu_util import to_padded
from oracle import post

B = 6
SAMPLE = [0, 4, 5]


@pytest.fixture(scope="module")
def small():
    W = plan.synth_weights("yolov8", 0, variant="n")
    pb = plan.build_yolov8(W, "n", in_h=96, in_w=128)
    x = np.concatenate([post.yolo_prepare_input(synth.frame(s), pb.in_h, pb.in_w)[0] for s in range(B)])
    bufs = pi.interpret(pb, to_padded(x.astype(np.float16).astype(np.float32), 4).astype(np.float64), B, round_to_plan=True)
    return pb, bufs


def test_subset_op_ref_equals_full_batch(small):
    pb, bufs = small
    sub = rc.subset(pb, bufs, SAMPLE)
    for i in range(len(pb.ops)):
        ref, bnd = pi.op_ref(pb, i, bufs, B)
        rs, bs = pi.op_ref(pb, i, sub, len(SAMPLE))
        assert np.array_equal(rs, ref[SAMPLE]), (i, pi.op_kind(pb, i))
        assert (bnd is None) == (bs is None) and (bnd is None or np.array_equal(bs, bnd[SAMPLE])), i
        assert np.array_equal(pi.read_out(pb, i, sub, len(SAMPLE)), pi.read_out(pb, i, bufs, B)[SAMPLE]), i


def test_clean_buffers_pass(small):
    pb, bufs = small
    worst = {}
    assert rc.check_images(pb, rc.subset(pb, bufs, SAMPLE), SAMPLE, set(pi.stale_reads(pb)), worst) == []
    assert max(worst.values()) < 1.0


def test_error_in_one_element_is_located(small):
    """A few bounds of error in one element of image 5 of a 3x3 conv's output: reported first with that op and image 5, and with
    no other image (ops reading the changed element may follow)"""
    pb, bufs = small
    i = [j for j in range(len(pb.ops)) if pi.op_kind(pb, j) == "gemm-9tap"][len(pb.ops) // 8]
    ref, bnd = pi.op_ref(pb, i, bufs, B)
    got = pi.read_out(pb, i, bufs, B)
    e = np.unravel_index(np.argmax(bnd[5]), bnd[5].shape)
    bad = {k: v.copy() for k, v in bufs.items()}
    got[(5,) + e] = ref[(5,) + e] + 4 * bnd[(5,) + e]
    pi.write_out(pb, i, bad, B, got)
    fails = rc.check_images(pb, rc.subset(pb, bad, SAMPLE), SAMPLE, set(pi.stale_reads(pb)), {})
    assert fails and fails[0][:3] == (i, "gemm-9tap", 5) and fails[0][3] == 1, fails[:3]
    assert {f[2] for f in fails} == {5}


def test_swapped_images_are_reported_by_digests(small):
    pb, bufs = small
    first = rc.stream_read(pb, lambda i: bufs[i], B, SAMPLE)
    assert first.halo == []
    k = max(range(len(pb.buffers)), key=lambda j: pb.buffers[j][0] * pb.buffers[j][1])
    rows = pb.buffers[k][0]
    bad = dict(bufs)
    bad[k] = bufs[k].copy()
    bad[k][rows:2 * rows], bad[k][2 * rows:3 * rows] = bufs[k][2 * rows:3 * rows], bufs[k][rows:2 * rows]
    again = rc.stream_read(pb, lambda i: bad[i], B, SAMPLE)
    assert rc.digest_diff(first.digests, again.digests) == [(k, 1), (k, 2)]
    assert rc.digest_diff({k: first.digests[k]}, {k: again.digests[k]}, [1, 2], [2, 1]) == []     # the same rows, swapped
    assert all(np.array_equal(first.sampled[j], again.sampled[j]) for j in bufs)  # the sampled images 0, 4, 5 are untouched
    assert np.array_equal(first.sampled[k], rc.subset(pb, bufs, SAMPLE)[k])


def test_halo_fault_is_reported(small):
    pb, bufs = small
    k = next(j for j, b in enumerate(pb.buffers) if b[3] > 0 and j != pb.image.buf)
    bad = dict(bufs)
    bad[k] = bufs[k].copy()
    bad[k][5 * pb.buffers[k][0] + pb.buffers[k][0] - 1, 0] = 1.0              # image 5, last halo row, last column
    assert rc.stream_read(pb, lambda i: bad[i], B, SAMPLE).halo == [k]


def test_schedule_reaches_every_case():
    s, win = rc.SCHEDULE, rc.windows(rc.SCHEDULE)
    cams = rc.rig_cameras()
    assert len(cams) == 8
    multi = [(g, w) for (kind, g, _), w in zip(s, win) if kind == "multi"]
    leads = {g[0] for g, _ in multi if len(g) > 1}
    assert any(g == rc.ALL for g, _ in multi)
    assert any(len(g) == 1 for g, _ in multi)                                        # K = 1 through update_multi
    assert any(len(g) > 1 and tuple(reversed(g)) in [h for h, _ in multi[:k]] for k, (g, _) in enumerate(multi))
    # a lead that has never touched the device, with a camera of more than 120 rows behind it
    fresh_crowd = False
    for k, ((kind, g, _), w) in enumerate(zip(s, win)):
        seen = {c for _, h, _ in s[:k] for c in h}
        if kind == "multi" and len(g) > 1 and g[0] not in seen and max(len(rc.stream_frame(cams, g[1], f)[1]) for f in w[g[1]]) > 120:
            fresh_crowd = True
    assert fresh_crowd
    # plain update and update_batch on trackers that lead other groups
    assert {g[0] for kind, g, _ in s if kind == "update"} & leads and {g[0] for kind, g, _ in s if kind == "batch"} & leads
    # a lead whose first call is small (one camera of a few objects) and that later leads a call whose association rows pass the
    # staging's minimum sizes (65536 cost entries; once a crowd is tracked its pool is about its detection count)
    grows = False
    for c in leads | {g[0] for g, _ in multi}:
        calls = [(g, w) for g, w in multi if g[0] == c]
        first = next((g, w) for (_, g, _), w in zip(s, win) if c in g)
        small = first[0] == (c,) and max(len(rc.stream_frame(cams, c, f)[1]) for f in first[1][c]) < 32
        later = any(sum(max(rc.high_dets(cams, d, f) for f in w[d]) ** 2 for d in g) > 65536 for g, w in calls[1:])
        grows |= small and later
    assert grows
    assert all(n >= 1 for _, _, n in s) and all(kind in ("multi", "update", "batch") for kind, _, _ in s)
    assert all(n == 1 for kind, _, n in s if kind == "update") and all(len(g) == 1 for kind, g, _ in s if kind != "multi")
    assert all(len(set(g)) == len(g) for _, g, _ in s)
