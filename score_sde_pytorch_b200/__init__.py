"""score_sde_pytorch_b200 — predictor–corrector sampling engine for the H100 (sm_90a) with the
sampling surface of yang-song/score_sde_pytorch (``sampling``, ``sde_lib``, ``models.utils``,
``models.ncsnpp``, ``op``).  See README.md / INTEGRATION.md."""
from . import configs, sde_lib   # noqa: F401
from . import models             # noqa: F401  (registers 'ncsnpp')
from . import sampling           # noqa: F401

__version__ = '0.1.0'
