"""Score models.  Importing the package registers ``'ncsnpp'`` and ``'ddpm'`` (``models/utils.register_model``)."""
from . import utils
from . import ncsnpp
from . import ddpm
