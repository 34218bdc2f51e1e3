"""uncalled_b200: H100-native implementation of the `uncalled map` hot path
(skovaka/UNCALLED) behind a C-ABI (include/unc_b200.h)."""
from ._native import UncError, build, default_params  # noqa: F401
from .mapper import BatchMapper, Index, make_descs, paf_key  # noqa: F401
from .stream import StreamMapper, feed_reads  # noqa: F401
from .index import BwaIndex, index_cmd, self_align  # noqa: F401
from .mask import mask_external, mask_internal  # noqa: F401
from .repeats import RepeatFinder  # noqa: F401

__version__ = "0.1.0"
from .dtw import (DTW_EVENT_GLOB, DTW_EVENT_QSUB, DTW_EVENT_RSUB, DTW_RAW_GLOB, DTW_RAW_QSUB, DTW_RAW_RSUB,  # noqa: F401
                  DTWParams, DTWr94d, DTWr94p, DTWSubSeq, dtw_batch)
from .signal import EventBatch, SignalProcessor, annotate, detect_events, match_probs, normalize  # noqa: F401
