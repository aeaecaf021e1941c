"""CPU oracle for the keras-ocr ``Pipeline.recognize`` hot path.

TEST INFRASTRUCTURE ONLY.  Nothing under ``oracle/`` is imported by the product
package (``keras-ocr_b200/``).  Only ``tests/``, ``__graft_entry__.smoke()`` and
``bench.py``'s ``cpu_baseline`` / ``--impl reference`` legs may import it, and
only as the checker / the CPU baseline.

Every function restates one piece of the reference (keras-ocr,
faustomorales/keras-ocr @ 9661d6f) and cites the file:line it follows.  The
restatement is validated in the authoring container against the reference's own
code by ``oracle/validate_against_reference.py`` (which AST-lifts the reference
functions at run time -- nothing is copied) and pinned by the fixtures that
script writes to ``tests/golden/``.

Pinning status (see DESIGN.md, "Oracle"):

* CRAFT graph            -- pinned: equals the reference's own PyTorch twin
                            (detection.py:472-644) to 1e-5 on seeded weights, and the
                            reference's Keras graph (build_keras_model +
                            load_torch_weights source, detection.py:65-103, 290-468,
                            executed on oracle/keras_shim.py) to 1.2e-5.
* getBoxes / warpBox /
  resize / pad / inputs  -- pinned: equal to the lifted reference functions
                            (same OpenCV 4.13) on the golden cases.
* CRNN + STN + CTC       -- PARTLY pinned.  TensorFlow is not installable here, but
                            the reference's own source of ``build_model``,
                            ``_transform`` and ``CTCDecoder`` (recognition.py:54-350)
                            is executed on ``oracle/keras_shim.py`` (numpy ``tf`` ops,
                            torch-backed Keras layers): graph wiring, the STN sampler
                            line by line and the CTC padding equal the restatement
                            (softmax to 4e-7, labels identical; tests/golden/crnn.npz).
                            The arithmetic INSIDE each Keras layer (Conv2D, BN eps 1e-3,
                            LSTM gates i,f,c,o, greedy ctc_decode) follows the Keras
                            documentation (SURVEY.md App. B) and stays UNPINNED
                            against TensorFlow's kernels.
* shapely                -- absent; ``minimum_rotated_rectangle`` is restated
                            as identity on 4-corner rectangles (the reference's
                            own AttributeError fallback, tools.py:548-550).
"""
