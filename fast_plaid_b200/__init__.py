"""fast_plaid_b200 -- an H100-native (sm_90a) PLAID search engine behind the FastPlaid surface.

    from fast_plaid_b200 import search
    index = search.FastPlaid(index="my_index", device="cuda:0")
    index.create(documents_embeddings)          # same on-disk layout as lightonai/fast-plaid
    index.search(queries_embeddings, top_k=10)  # -> list[list[(doc_id, score)]]
"""

from . import search  # noqa: F401

__version__ = "0.1.0"
__all__ = ["search"]
