"""kafka_topic_analyzer_b200 — H100-native (sm_90a) message-scan metric aggregation for
kafka-topic-analyzer: the per-record path of src/kafka.rs:92-135 → src/metric.rs:206-305 →
src/fnv32.rs:92-101, rebuilt as hand-written CUDA behind a C ABI (include/kta.h).

Layout: csrc/ (CUDA kernels + the C ABI), _native.py (ctypes loader + nvcc recipe),
metrics.py (host mirror of the reference's MetricHandler / MessageMetrics interface),
synth.py (the synthetic in-memory topic).  No CPU fallback exists in this package.
"""
from ._native import KtaError, build, lib  # noqa: F401
from .metrics import (KtaEngine, LogCompactionInMemoryMetrics, Message, MessageMetrics,  # noqa: F401
                      TopicAnalyzer)

__version__ = "0.1.0"
