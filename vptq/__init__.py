"""Drop-in alias: `from vptq import VQuantLinear` / `import vptq.ops` resolve to vptq_b200.

Hugging Face transformers imports the quantized layer as `from vptq import VQuantLinear`
(transformers/integrations/vptq.py); putting this repository on sys.path makes that import land
on the H100 implementation without touching transformers.
"""
import sys

import vptq_b200
from vptq_b200 import VQuantLinear, __version__, ops

sys.modules[__name__ + ".ops"] = ops
sys.modules[__name__ + ".layers"] = vptq_b200.layers

__all__ = ["VQuantLinear", "ops", "__version__"]
