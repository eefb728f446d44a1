from ._functions import (GroupedMatMul4Bit, GroupedMatMul8bitLt, MatMul4Bit, MatMul8bitLt,  # noqa: F401
                         MatmulLtState, grouped_matmul_4bit, grouped_matmul_8bit, matmul, matmul_4bit)
