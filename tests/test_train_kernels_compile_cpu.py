"""CPU: the training kernels compile without a stack frame or spills.

The GEMM kernels of csrc/train.cu share force-inlined helpers that take the shared tiles and the accumulator
by reference.  Once inlined they cost nothing; a helper that ptxas cannot keep in registers puts the
accumulator on the stack instead, and nothing fails then: results stay the same and only the kernel slows
down.  So this compiles train.cu with the library's flags and reads ptxas's resource report for every
training kernel.  Skipped when no nvcc is installed.
"""
from toolchain import compile_cuda, kernel_key

KERNELS = [
    "train_fwd_kernel<false>", "train_fwd_finish_kernel<false>", "train_reduce_kernel<false>", "train_dw_kernel<false>",
    "train_dx_kernel<false>", "train_pool_fwd_kernel", "train_pool_bwd_kernel", "train_finalize_kernel",
    "train_adam_kernel", "train_fwd_plain_kernel<false>", "train_dx_plain_kernel", "train_dw_plain_kernel<false>",
]


def test_train_kernels_no_stack_no_spills():
    by_name = {kernel_key(m): k.local_memory for m, k in compile_cuda("train.cu").kernels.items() if kernel_key(m)}
    missing = [k for k in KERNELS if k not in by_name]
    assert not missing, "kernels not compiled: %s (found %s)" % (missing, sorted(by_name))
    for k in KERNELS:
        assert by_name[k] == (0, 0, 0), "%s: %d-byte stack frame, %d / %d bytes spilled (stores / loads)" % (
            (k,) + by_name[k])
