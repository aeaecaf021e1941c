"""Plain NumPy references for reading words in quarter turns: the crop in turn r (``b2o_warp_boxes_turned``) and the
vote between the turns' readings (``b2o_select_rotation``), with the crafted vote cases the GPU tests run.

Turn r cuts ``warpBox(image, np.roll(c, -r, axis=0), 31, 200, skip_rotate=True)`` with c = ``order_corners(box)``:
the plan is built from the same pinned pieces as ``image_refs.warp_transform`` (the order, ``rotated_width_height``,
``cvmodels.get_persp`` / ``inv3``), with the roll between the order and the measurement, and sampled by
``image_refs.warp_sample``.  tests/test_rotation_refs.py pins both against cv2 and the vote on crafted arrays."""
import numpy as np

from tests import cvmodels as M
from tests import image_refs as IR

STEPS = 48


def turned_box(quad, r):
    """np.roll(order_corners(quad), -r, axis=0): the box warpBox cuts in turn r, float32 (4,2)."""
    from oracle import imageops
    return np.roll(imageops.order_corners(quad), -int(r), axis=0)


def turned_transform(quad, r, target_w=IR.CROP_W, target_h=IR.CROP_H):
    """(forward M (3,3), dw, dh) of warpBox(skip_rotate=True) on the turned box; ZeroDivisionError where w or h is 0."""
    from oracle import imageops
    box = turned_box(quad, r)
    w, h = imageops.rotated_width_height(box)
    scale = min(target_w / w, target_h / h)
    dst = np.array([[0, 0], [scale * w, 0], [scale * w, scale * h], [0, scale * h]]).astype("float32")
    return M.get_persp(box, dst), int(scale * w), int(scale * h)


def turned_warp(img, quad, r):
    """(crop (31,200[,C]) uint8, plan (m, dw, dh) or None) of turn r; an all-zero crop where warpBox raises
    ZeroDivisionError, as ``image_refs.warp_box``."""
    try:
        fwd, dw, dh = turned_transform(quad, r)
    except ZeroDivisionError:
        return np.zeros((IR.CROP_H, IR.CROP_W) + img.shape[2:], np.uint8), None
    plan = (M.inv3(fwd).reshape(-1), dw, dh)
    return IR.warp_sample(img, *plan), plan


def select(labels, logp, image_index, turns, vote, boxes=None):
    """The vote of ``b2o_select_rotation``.  labels (R,b,P,48), logp (R,b,P) in the order of ``turns``; image_index (b)
    non-decreasing.  "word": per word the slot with the largest logp[j,k,0]; "page": per image the slot with the
    largest float32 sum of logp[j,k,0] over its words in word order.  Strictly larger wins, so ties and all -inf keep
    the first listed turn.  Returns (labels (b,P,48), logp (b,P), turns (b,) int32, rolled boxes (b,4,2) or None)."""
    labels, logp = np.asarray(labels), np.asarray(logp, np.float32)
    r, b = logp.shape[:2]
    best = logp[:, :, 0]
    pick = np.zeros(b, np.int64)
    if vote == "word":
        for k in range(b):
            for j in range(1, r):
                if best[j, k] > best[pick[k], k]:
                    pick[k] = j
    else:
        for img in np.unique(image_index):
            ks = np.flatnonzero(np.asarray(image_index) == img)
            sums = []
            for j in range(r):
                s = np.float32(0)
                for k in ks:
                    s = np.float32(s + best[j, k])
                sums.append(s)
            p = 0
            for j in range(1, r):
                if sums[j] > sums[p]:
                    p = j
            pick[ks] = p
    rows = np.arange(b)
    chosen = np.asarray(turns, np.int32)[pick]
    rolled = None
    if boxes is not None:
        rolled = np.stack([turned_box(q, t) for q, t in zip(boxes, chosen)]) if b else np.zeros((0, 4, 2), np.float32)
    return labels[pick, rows], logp[pick, rows], chosen, rolled


def _rect(rng, w_img=400, h_img=300):
    return IR._rect(rng.uniform(0, w_img), rng.uniform(0, h_img), rng.uniform(8, 160), rng.uniform(4, 40),
                    rng.uniform(-90, 90), int(rng.integers(4)), bool(rng.integers(2)))


def select_cases(seed=0):
    """Crafted inputs for the vote: dicts of name, labels (R,b,P,48) int32, logp (R,b,P) float32, image_index (b) int32,
    n_images, turns, boxes (b,4,2) float32.  They have exact ties between turns, -inf rows (one turn or all), images
    without words (at the start, inside and at the end), P = 1 / 3 / 128, R = 1 ... 4 and turn lists in other than
    ascending order."""
    rng = np.random.default_rng(seed)
    cases = []

    def add(name, turns, counts, p, tie=0.3, ninf=0.1):
        r, b = len(turns), int(sum(counts))
        logp = -rng.exponential(3.0, (r, b, p)).astype(np.float32)
        logp = -np.sort(-logp, axis=2)                     # best first, as the decoders write them
        for k in range(b):
            u = rng.random()
            if u < tie and r > 1:                          # an exact tie between two turns on the best reading
                j0, j1 = rng.choice(r, 2, replace=False)
                logp[j1, k, 0] = logp[j0, k, 0]
            elif u < tie + ninf:                           # -inf rows: one turn, or every turn
                js = range(r) if rng.random() < 0.5 else [int(rng.integers(r))]
                for j in js:
                    logp[j, k, :] = -np.inf
        labels = rng.integers(-1, 37, (r, b, p, STEPS)).astype(np.int32)
        index = np.repeat(np.arange(len(counts), dtype=np.int32), counts)
        boxes = np.stack([_rect(rng) for _ in range(b)]).astype(np.float32) if b else np.zeros((0, 4, 2), np.float32)
        cases.append(dict(name=name, labels=labels, logp=np.ascontiguousarray(logp), image_index=index,
                          n_images=len(counts), turns=tuple(turns), boxes=boxes))

    add("R1_P1", (0,), [3, 0, 5], 1)
    add("R2_P1_upside_down", (0, 2), [0, 7, 4, 0, 9], 1)
    add("R4_P1", (0, 1, 2, 3), [12, 1, 0, 30, 2], 1)
    add("R4_P1_ties_everywhere", (0, 1, 2, 3), [6, 6], 1, tie=0.9, ninf=0.05)
    add("R3_P3_order_2_0_3", (2, 0, 3), [5, 0, 11], 3)
    add("R4_P128_order_3_1_0_2", (3, 1, 0, 2), [2, 3, 0], 128)
    add("R2_P1_all_inf", (1, 3), [4, 4], 1, tie=0.0, ninf=1.0)
    add("R4_P1_long_page", (0, 1, 2, 3), [0, 257], 1)
    # whole images whose every word ties, or is -inf in every turn: the page keeps the first listed turn
    r, b = 3, 6
    logp = np.full((r, b, 1), -2.5, np.float32)
    logp[:, 3:] = -np.inf
    cases.append(dict(name="R3_pages_tie_and_inf", labels=rng.integers(-1, 37, (r, b, 1, STEPS)).astype(np.int32),
                      logp=logp, image_index=np.array([0, 0, 0, 2, 2, 2], np.int32), n_images=3, turns=(1, 2, 0),
                      boxes=np.stack([_rect(rng) for _ in range(b)]).astype(np.float32)))
    return cases
