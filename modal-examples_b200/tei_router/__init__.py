"""In-box stand-in for Hugging Face text-embeddings-inference's ``text-embeddings-router`` (Face 2 of the
drop-in boundary, SURVEY.md §2.3): same executable name, flags, TCP-readiness semantics and ``POST /embed``
contract as the TEI 1.7 server the reference launches at
``06_gpu_and_ml/embeddings/text_embeddings_inference.py:29-51`` and calls at ``:100``; the arithmetic runs on the
local H100s through ``b200rt``."""
