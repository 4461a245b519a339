"""youtokentome_b200 — H100-native BPE trainer / encoder with the YouTokenToMe surface.

    import youtokentome_b200 as yttm
    yttm.BPE.train(data="train.txt", model="m.yttm", vocab_size=5000)
    bpe = yttm.BPE(model="m.yttm")
    bpe.encode(["some text"], output_type=yttm.OutputType.ID)

Both hot paths (training merge loop, batch encode) run as sm_90a CUDA kernels behind the C ABI
in include/yttm_b200.h; there is no CPU fallback.
"""
from .youtokentome import BPE, OutputType, WordCounts, release_training_cache, train_report  # noqa: F401

__all__ = ["BPE", "OutputType", "WordCounts", "release_training_cache", "train_report"]
