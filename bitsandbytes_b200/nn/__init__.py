from .embedding import (  # noqa: F401
    Embedding,
    Embedding4bit,
    Embedding8bit,
    EmbeddingFP4,
    EmbeddingNF4,
    StableEmbedding,
)
from .modules import (  # noqa: F401
    GroupedLinear4bit,
    GroupedLinear8bitLt,
    Int8Params,
    Linear4bit,
    Linear8bitLt,
    LinearFP4,
    LinearNF4,
    Params4bit,
    fix_4bit_weight_quant_state_from_module,
)
from . import parametrize  # noqa: F401
