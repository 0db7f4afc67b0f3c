"""Drop-in shim: put this directory first on PYTHONPATH and the reference's `train.py` / `predict.py`
(`from mtad_gat import MTAD_GAT`, train.py:7 / predict.py:7) resolve to the H100 implementation."""
from mtad_gat_pytorch_b200.mtad_gat import MTAD_GAT  # noqa: F401
