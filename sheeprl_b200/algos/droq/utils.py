"""DroQ side constants the CLI looks up in `<algo module>.utils` (sheeprl/cli.py:151-181; reference:
sheeprl/algos/droq/utils.py:17-18, SAC's)."""
from sheeprl_b200.algos.sac.utils import AGGREGATOR_KEYS, MODELS_TO_REGISTER  # noqa: F401
