"""The reference's ``custommodels`` package (biencoder/beir/custommodels/__init__.py) on this library's CUDA kernels."""
from sgpt_b200.embedder import SentenceBERTAsym, SentenceBERTBOSEOS  # noqa: F401
from sgpt_b200.exact_search import DenseRetrievalExactSearch  # noqa: F401
