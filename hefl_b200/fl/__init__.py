"""Federated-learning runtime: data, local training, round loop, checkpoints."""
from .runner import FederatedRunner, classification_metrics, simulate_clients  # noqa: F401
from .server_opt import SERVER_OPTS, ServerOptimizer, check_server_options  # noqa: F401
from .trainer import LocalTrainer  # noqa: F401
