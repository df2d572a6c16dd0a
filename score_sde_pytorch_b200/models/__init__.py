"""Score models.  Importing the package registers ``'ncsnpp'``, ``'ddpm'``, ``'ncsnv2_64'`` and ``'ncsnv2_128'`` (``models/utils.register_model``)."""
from . import utils
from . import ncsnpp
from . import ddpm
from . import ncsnv2
