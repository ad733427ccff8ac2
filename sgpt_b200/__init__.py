"""sgpt_b200 — H100-native (sm_90a) SGPT bi-encoder hot path (GPT forward -> weighted-mean pool -> cosine/dot top-k).

Public surface mirrors the reference's plug-in protocols (biencoder/beir/beir_dense_retriever.py,
biencoder/beir/custommodels/exact_search.py):

    from sgpt_b200 import CustomEmbedder, DenseRetrievalExactSearch
    model = DenseRetrievalExactSearch(CustomEmbedder(model_name, method="weightedmean", specb=True), batch_size=128)
    results = model.search(corpus, queries, top_k=1000, score_function="cos_sim")

All arithmetic runs in the in-tree CUDA library (libsgpt_b200.so, sm_90a: H100); importing the package does not load it,
using it without the library raises.
"""
from .config import ModelConfig, preset  # noqa: F401

__all__ = ["ModelConfig", "preset", "Encoder", "CustomEmbedder", "SentenceEncoder", "SentenceBERTBOSEOS",
           "SentenceBERTAsym", "DenseRetrievalExactSearch", "CorpusShard", "merge_topk", "semantic_search",
           "merge_topk_packed", "unpack_topk", "pack_mask", "IVFIndex", "IVFPQIndex", "GraphIndex", "sharded_search", "PeerGather", "ShardedDenseRetrievalExactSearch", "DenseHead", "AsymHeads", "load_st_directory", "GenericDataLoader", "EvaluateRetrieval",
           "InformationRetrievalEvaluator", "paraphrase_mining", "paraphrase_mining_embeddings", "community_detection"]


def __getattr__(name):  # lazy: torch / CUDA pieces are imported on first use
    if name == "Encoder":
        from .encoder import Encoder
        return Encoder
    if name in ("DenseHead", "AsymHeads"):
        from . import heads
        return getattr(heads, name)
    if name == "load_st_directory":
        from .st_loader import load_st_directory
        return load_st_directory
    if name == "InformationRetrievalEvaluator":
        from .evaluation import InformationRetrievalEvaluator
        return InformationRetrievalEvaluator
    if name in ("GenericDataLoader", "EvaluateRetrieval"):
        from . import beir_compat
        return getattr(beir_compat, name)
    if name in ("CustomEmbedder", "SentenceEncoder", "SentenceBERTBOSEOS", "SentenceBERTAsym"):
        from . import embedder
        return getattr(embedder, name)
    if name == "DenseRetrievalExactSearch":
        from .exact_search import DenseRetrievalExactSearch
        return DenseRetrievalExactSearch
    if name in ("CorpusShard", "merge_topk", "merge_topk_packed", "unpack_topk", "pack_mask", "semantic_search"):
        from . import index
        return getattr(index, name)
    if name == "IVFIndex":
        from .ivf import IVFIndex
        return IVFIndex
    if name == "IVFPQIndex":
        from .ivfpq import IVFPQIndex
        return IVFPQIndex
    if name == "GraphIndex":
        from .graph import GraphIndex
        return GraphIndex
    if name in ("paraphrase_mining", "paraphrase_mining_embeddings", "community_detection"):
        from . import mining
        return getattr(mining, name)
    if name in ("sharded_search", "PeerGather", "ShardedDenseRetrievalExactSearch"):
        from . import dist
        return getattr(dist, name)
    raise AttributeError(name)
