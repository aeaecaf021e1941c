"""keras-ocr_b200: an H100-native drop-in for ``keras_ocr.pipeline.Pipeline.recognize``.

Public surface mirrors the reference (keras_ocr/pipeline.py:7-75, detection.py:661-785,
recognition.py:353-537): ``Pipeline``, ``Detector``, ``Recognizer``.  Every stage runs as a
hand-written sm_90a CUDA kernel behind the C-ABI in ``include/b2ocr.h``; there is no CPU
fallback -- importing the compute classes without the built library raises.
"""
__version__ = "0.1.0"

from . import weights  # noqa: F401  (pure numpy, importable without the CUDA library)


def __getattr__(name):
    # Lazy so that `import keras_ocr_b200.weights` works on machines without the built .so.
    if name in ("Pipeline", "Detector", "Recognizer"):
        from . import pipeline, detection, recognition
        return {"Pipeline": pipeline.Pipeline, "Detector": detection.Detector,
                "Recognizer": recognition.Recognizer}[name]
    raise AttributeError(name)
