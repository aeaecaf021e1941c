"""CPU: the host side of detection scores and word confidences -- the scored record layout, its multi-process gather
(gloo, world size 2), the refusal of injected components, and the oracle's box scores."""
import os
import socket

import cv2
import numpy as np
import pytest
import torch.distributed as dist
import torch.multiprocessing as mp

from keras_ocr_b200 import distributed as D, recognition
from tests import score_refs

ALPHABET = "0123456789abcdefghijklmnopqrstuvwxyz"


def _random_block(rng, counts, per_rank, max_boxes):
    boxes = [rng.uniform(0, 900, (c, 4, 2)).astype(np.float32) for c in counts]
    labels = rng.integers(-1, 37, (sum(counts), 48)).astype(np.int8)
    box_scores = [rng.uniform(0.7, 1.0, c).astype(np.float32) for c in counts]
    logp = -rng.exponential(2.0, sum(counts)).astype(np.float32)
    return boxes, labels, box_scores, logp


def test_scored_records_roundtrip_and_unscored_prefix():
    rng = np.random.default_rng(3)
    blocks, plain, expect = [], [], []
    for per_rank, counts in ((3, [2, 0, 8]), (3, [1, 5])):      # second block: a short shard (one padding row)
        boxes, labels, box_scores, logp = _random_block(rng, counts, per_rank, 8)
        scored = D.pack_records(counts, boxes, labels, per_rank, 8, box_scores=box_scores, logp=logp)
        unscored = D.pack_records(counts, boxes, labels, per_rank, 8)
        assert scored.shape == (per_rank, D.record_floats(8, scores=True)) == (per_rank, 1 + 8 * 8 + 8 * 12 + 16)
        # the unscored record is a prefix of the scored one, bit for bit
        assert np.array_equal(scored.numpy()[:, :D.record_floats(8)].view(np.int32), unscored.numpy().view(np.int32))
        blocks.append(scored)
        plain.append(unscored)
        expect.append((counts, boxes, labels, box_scores, logp))
    counts, boxes, labels, sc, lp = D.unpack_blocks(blocks, 8, scores=True)
    assert counts.tolist() == [2, 0, 8, 1, 5]
    assert np.array_equal(boxes, np.concatenate([b for e in expect for b in e[1]]))
    assert np.array_equal(labels, np.concatenate([e[2] for e in expect]))
    assert np.array_equal(sc, np.concatenate([s for e in expect for s in e[3]]))
    assert np.array_equal(lp, np.concatenate([e[4] for e in expect]))
    c2, b2, l2 = D.unpack_blocks(plain, 8)                      # the unscored reader is untouched
    assert np.array_equal(c2, counts) and np.array_equal(b2, boxes) and np.array_equal(l2, labels)


def test_confidences_are_clipped_exponentials():
    s = np.array([-30.0, -1.0, 0.0, 48 * np.log1p(1e-7)], np.float32)
    c = recognition.confidences(s)
    assert c.dtype == np.float32 and np.all(c > 0) and np.all(c <= 1)
    assert np.array_equal(c[:3], np.exp(s[:3]))


# ---------------------------------------------------------------------------- gather with scores, world size 2
class _Stage:
    device = None
    alphabet = ALPHABET


class _ScoredPipeline:
    """Two-phase records pipeline (like the real Pipeline) whose words, detection scores and log-probabilities are a
    deterministic function of the image content, built with the host ``pack_records``."""
    detector = _Stage()
    recognizer = _Stage()

    @staticmethod
    def words(images):
        out = []
        for im in images:
            v = int(im[0, 0, 0])
            out.append([(ALPHABET[(v + j) % 36] * (1 + j), np.full((4, 2), v + 0.25 * j, np.float32),
                         np.float32(0.7 + 0.01 * v + 0.001 * j), np.float32(-0.1 * v - 0.5 * j)) for j in range(v % 4)])
        return out

    def expected(self, images):
        return [[(t, b.tolist(), float(s), float(recognition.confidences([lp])[0])) for t, b, s, lp in g]
                for g in self.words(images)]

    def records_begin(self, images, rows=None, rec_boxes=128, scores=False):
        return {"images": images, "rows": rows, "rec_boxes": rec_boxes, "scores": scores}

    def records_counts(self, state):
        return [len(g) for g in self.words(state["images"])]

    def records_end(self, state, rec_boxes=None):
        assert state["scores"]
        g = self.words(state["images"])
        labels = np.full((sum(len(x) for x in g), 48), -1, np.int8)
        k = 0
        for words in g:
            for text, *_ in words:
                labels[k, :len(text)] = [ALPHABET.index(ch) for ch in text]
                k += 1
        return D.pack_records([len(x) for x in g], [np.array([w[1] for w in x], np.float32).reshape(-1, 4, 2) for x in g],
                              labels, state["rows"], state["rec_boxes"] if rec_boxes is None else rec_boxes,
                              box_scores=[np.array([w[2] for w in x], np.float32) for x in g],
                              logp=np.array([w[3] for x in g for w in x], np.float32))

    def recognize_records(self, images, rows=None, rec_boxes=128, scores=False):
        return self.records_end(self.records_begin(images, rows, rec_boxes, scores))


def _plain(result):
    return [[(t, np.asarray(b).tolist(), float(s), float(c)) for t, b, s, c in g] for g in result]


def _worker(rank, world, port, images, batches, ret):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        pipe = _ScoredPipeline()
        sharded = D.recognize_sharded(pipe, images, max_boxes=8, return_scores=True)
        auto = D.recognize_sharded(pipe, images, max_boxes="auto", return_scores=True)
        stream = D.ShardedStream(pipe, max_boxes=8, return_scores=True)
        outs = [stream.submit(b[rank * 2:(rank + 1) * 2]) for b in batches]
        outs.append(stream.flush())
        if rank == 0:
            ret.put((_plain(sharded), _plain(auto), [None if o is None else _plain(o) for o in outs]))
        else:
            assert sharded is None and auto is None and all(o is None for o in outs)
    finally:
        dist.destroy_process_group()


def test_scored_gather_world2_gloo():
    images = np.zeros((7, 4, 4, 3), np.uint8)
    images[:, 0, 0, 0] = np.arange(7) + 1
    batches = []
    for k in range(3):
        im = np.zeros((4, 4, 4, 3), np.uint8)
        im[:, 0, 0, 0] = np.arange(4) + 1 + 4 * k
        batches.append(im)
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    ctx = mp.get_context("spawn")
    ret = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, images, batches, ret)) for r in range(2)]
    for p in procs:
        p.start()
    sharded, auto, streamed = ret.get(timeout=120)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    pipe = _ScoredPipeline()
    assert sharded == auto == pipe.expected(images)          # global order, words, scores: bit for bit
    assert sum(len(g) for g in sharded) > 0
    assert streamed[0] is None and streamed[1:] == [pipe.expected(b) for b in batches]


# ---------------------------------------------------------------------------- injected components
class _DuckDetector:
    def detect(self, images, **kw):
        return [np.zeros((0, 4, 2), np.float32) for _ in images]


class _DuckRecognizer:
    alphabet = ALPHABET

    def recognize_from_boxes(self, images, box_groups, **kw):
        return [[] for _ in images]


def test_return_scores_with_injected_components_raises():
    from keras_ocr_b200.pipeline import Pipeline
    pipe = Pipeline(detector=_DuckDetector(), recognizer=_DuckRecognizer())
    images = np.full((1, 40, 40, 3), 255, np.uint8)
    assert pipe.recognize(images) == [[]]                     # the default call is served as before
    with pytest.raises(NotImplementedError, match="injected"):
        pipe.recognize(images, return_scores=True)
    with pytest.raises(NotImplementedError):
        D.recognize_sharded(pipe, images, return_scores=True)
    with pytest.raises(NotImplementedError):
        D.ShardedStream(pipe, return_scores=True)


# ---------------------------------------------------------------------------- oracle box scores
def _component_maxima(scores, detection_threshold=0.7, text_threshold=0.4, link_threshold=0.4, size_threshold=10):
    """Independent restatement: the kept components of cv2.connectedComponentsWithStats in label order, and the
    largest text score over each."""
    text, link = scores[..., 0], scores[..., 1]
    union = ((text > text_threshold) | (link > link_threshold)).astype(np.uint8)
    count, labels, stats, _ = cv2.connectedComponentsWithStats(union, connectivity=4)
    out = []
    for cid in range(1, count):
        if stats[cid, cv2.CC_STAT_AREA] < size_threshold:
            continue
        m = np.max(np.where(labels == cid, text, -np.inf))
        if m >= detection_threshold:
            out.append(m)
    return np.array(out, np.float32)


@pytest.mark.parametrize("tag", ["grid32", "rot12", "dense", "blank", "refmaps"])
@pytest.mark.parametrize("thr", [0.7, 0.5, 0.9])
def test_oracle_box_scores_equal_component_maxima(golden_dir, tag, thr):
    from oracle import imageops
    g = np.load(os.path.join(golden_dir, "boxes.npz"))
    for scores in g[f"boxes_{tag}_scores"]:
        quads, sc = score_refs.box_scores(scores, detection_threshold=thr)
        assert len(sc) == len(quads)
        assert np.array_equal(sc, _component_maxima(scores, detection_threshold=thr))
        assert np.all(sc >= np.float32(thr))
        assert np.array_equal(quads, imageops.get_boxes_single(scores, detection_threshold=thr))
