"""numpy model of the box NMS on the device (k_post_nms, include/linemod_b200.h lm_enqueue_post / lm_complete_post),
and, kept apart from it, the reference drivers' own pipeline on a finished match list.

Records and matches are structured arrays with fields x, y, similarity, template_id and class_index (the native
library's) or class_idx (the oracle's).  Boxes are wh[g] = (width, height) of global template g = class_begin[c] + t.

Device semantics (the model):
  1. canonical order: similarity descending, then template_id, class, y, x ascending;
  2. canonical dedupe: drop each record equal in (x, y, similarity, class) to its predecessor in that order -- what
     std::unique (LL.cpp:1773, Match::operator== ignores template_id) removes from the sorted list;
  3. greedy NMS in that order (linemod_ros/detect.py:53, linemod_and_levelup_test.py:34-61): IoU in float64 with the
     "+1" pixel convention, a box is suppressed when ovr > thr;
  4. the first min(top_k, 1024) survivors (every survivor up to 1024 for top_k <= 0) come back;
     counts = [survivors written, raw records, survivors in total (top_k <= 0) or -1]."""
import numpy as np

POST_MAX = 1024


def _cls(a):
    return a["class_index"] if "class_index" in a.dtype.names else a["class_idx"]


def canonical_order(recs):
    return np.lexsort((recs["x"], recs["y"], _cls(recs), recs["template_id"], -recs["similarity"].astype(np.float64)))


def canonical_dedupe(recs):
    """The records std::sort + std::unique would keep, in canonical order."""
    s = recs[canonical_order(recs)]
    keep = np.ones(len(s), bool)
    if len(s) > 1:
        c = _cls(s)
        keep[1:] = ~((s["x"][1:] == s["x"][:-1]) & (s["y"][1:] == s["y"][:-1]) &
                     (s["similarity"][1:] == s["similarity"][:-1]) & (c[1:] == c[:-1]))
    return s[keep]


def boxes(dets, wh, class_begin):
    g = np.asarray(class_begin, np.int64)[_cls(dets).astype(np.int64)] + dets["template_id"].astype(np.int64)
    wh = np.asarray(wh, np.float64).reshape(-1, 2)[g].reshape(len(dets), 2)
    x1 = dets["x"].astype(np.float64)
    y1 = dets["y"].astype(np.float64)
    return x1, y1, x1 + wh[:, 0], y1 + wh[:, 1]


def greedy(dets, wh, class_begin, thr, want=None):
    """nms(dets, thr) of the drivers on dets taken in the order given: indices of the survivors, in pick order.
    Stops after `want` survivors when it is given."""
    x1, y1, x2, y2 = boxes(dets, wh, class_begin)
    areas = (x2 - x1 + 1) * (y2 - y1 + 1)
    order = np.arange(len(dets))
    keep = []
    while order.size > 0 and (want is None or len(keep) < want):
        i = order[0]
        keep.append(int(i))
        rest = order[1:]
        w = np.maximum(0.0, np.minimum(x2[i], x2[rest]) - np.maximum(x1[i], x1[rest]) + 1)
        h = np.maximum(0.0, np.minimum(y2[i], y2[rest]) - np.maximum(y1[i], y1[rest]) + 1)
        inter = w * h
        ovr = inter / (areas[i] + areas[rest] - inter)
        order = rest[ovr <= thr]
    return np.asarray(keep, np.int64)


def post_nms(records, wh, class_begin, thr, top_k=0):
    """The device's box NMS on the raw kept records (any order): (survivors in pick order, counts[3])."""
    d = canonical_dedupe(records)
    want = min(top_k, POST_MAX) if top_k > 0 else POST_MAX
    keep = greedy(d, wh, class_begin, thr, want if top_k > 0 else None)
    return d[keep[:want]], [int(min(len(keep), want)), len(records), -1 if top_k > 0 else len(keep)]


def raw_nms(records, wh, class_begin, thr):
    """The same greedy NMS without the dedupe (what the device did before it): survivors in pick order."""
    s = records[canonical_order(records)]
    return s[greedy(s, wh, class_begin, thr)]


def driver_nms(finished, wh, class_begin, thr):
    """The drivers' pipeline: nms() on the finished list (after the reference's std::sort + std::unique), equal
    similarities in the documented tie order."""
    s = finished[canonical_order(finished)]
    return s[greedy(s, wh, class_begin, thr)]


def same(a, b):
    return len(a) == len(b) and all(np.array_equal(a[f], b[f]) for f in ("x", "y", "similarity", "template_id")) and \
        np.array_equal(_cls(a), _cls(b))
