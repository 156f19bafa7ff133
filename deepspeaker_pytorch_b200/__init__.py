"""H100-native Deep Speaker hot path: drop-in for reference model.py's DeepSpeakerModel,
TripletMarginLoss and PairwiseDistance, backed by hand-written sm_90a CUDA behind a C ABI
(include/dsk.h, lib/libdsk.so)."""
from .model import (AAMSoftmaxLoss, BatchHardTripletLoss, DeepSpeakerModel, GE2ELoss, PairwiseDistance,  # noqa: F401
                    SupConLoss, TripletMarginLoss, allpairs_topk, select_hard_triplets)

from .pipeline import EmbeddingPipeline  # noqa: F401,E402
from .head import CrossEntropyLoss  # noqa: F401,E402
from .optim import FusedAdagrad  # noqa: F401,E402
from .steps import (aam_softmax_step, batch_hard_step, ge2e_step, sharded_aam_softmax_step, supcon_step,  # noqa: F401,E402
                    train_step)
from .parallel import (GlobalBatchHardTripletLoss, GlobalGE2ELoss, ShardedAAMSoftmaxLoss,  # noqa: F401,E402
                       class_shards)

__all__ = ["train_step", "batch_hard_step", "aam_softmax_step", "ge2e_step", "supcon_step", "CrossEntropyLoss",
           "FusedAdagrad", "EmbeddingPipeline", "DeepSpeakerModel", "PairwiseDistance", "TripletMarginLoss",
           "AAMSoftmaxLoss", "BatchHardTripletLoss", "GE2ELoss", "SupConLoss", "GlobalBatchHardTripletLoss",
           "GlobalGE2ELoss", "select_hard_triplets", "allpairs_topk", "ShardedAAMSoftmaxLoss", "class_shards",
           "sharded_aam_softmax_step"]
