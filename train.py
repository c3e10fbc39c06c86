"""Entry points `init_processes` / `run` of PipeGCN/train.py, implemented in pipegcn_b200.train."""
from pipegcn_b200.train import RankEngine, LocalTrainer, create_model, init_processes, run  # noqa: F401
