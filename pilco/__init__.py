"""Drop-in alias: ``import pilco`` resolves to the H100-native engine (``pilco_b200``), so the reference's
``tests/`` and ``examples/`` import lines (``from pilco.models import MGPR`` ...) work unchanged."""
import sys

import pilco_b200
from pilco_b200 import models, controllers, rewards   # noqa: F401
import pilco_b200.models.mgpr, pilco_b200.models.smgpr, pilco_b200.models.pilco   # noqa: F401,E401

sys.modules[__name__ + ".models"] = pilco_b200.models
sys.modules[__name__ + ".models.mgpr"] = pilco_b200.models.mgpr
sys.modules[__name__ + ".models.smgpr"] = pilco_b200.models.smgpr
sys.modules[__name__ + ".models.pilco"] = pilco_b200.models.pilco
sys.modules[__name__ + ".controllers"] = pilco_b200.controllers
sys.modules[__name__ + ".rewards"] = pilco_b200.rewards
