"""Import shim: makes `import bitsandbytes` resolve to bitsandbytes_b200, so that code written against the
reference package name (Hugging Face Transformers' bitsandbytes quantizer, PEFT) runs on the H100-native
implementation unchanged.  Put this directory's parent (`shim/`) in front of PYTHONPATH; the sibling
`bitsandbytes-0.50.2.dist-info` answers importlib.metadata's version query (Transformers requires
bitsandbytes >= 0.46.1) with the version of the reference snapshot whose API is mirrored."""
import sys

import bitsandbytes_b200 as _impl

sys.modules[__name__] = _impl
for _name in ("nn", "functional", "autograd", "utils", "optim"):
    _sub = getattr(_impl, _name, None)
    if _sub is not None:
        sys.modules[f"{__name__}.{_name}"] = _sub
