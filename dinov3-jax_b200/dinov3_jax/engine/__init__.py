from .config import EngineConfig, config_for, config_from_reference_cfg, distill_config_from_reference_cfg, from_oracle_cfg, ARCHS  # noqa: F401
from .core import Engine  # noqa: F401
