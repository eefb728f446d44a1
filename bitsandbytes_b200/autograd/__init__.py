from ._functions import (GroupedMatMul4Bit, MatMul4Bit, MatMul8bitLt, MatmulLtState,  # noqa: F401
                         grouped_matmul_4bit, matmul, matmul_4bit)
