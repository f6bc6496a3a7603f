"""Minimal stand-in for the un-vendored `arm_pytorch_utilities` dependency of the reference
(pyproject.toml:57), used ONLY by tests/golden/make_golden.py to import the live reference in
the build container.  Behaviour pinned by reference tests/test_batch_wrapper.py:19-47:
`handle_batch_input(n)` flattens extra leading batch dimensions so tensor arguments are n-D,
calls the function and restores the leading dimensions on the outputs."""
import functools
import torch


def handle_batch_input(n):
    def deco(fn):
        @functools.wraps(fn)
        def wrapped(*args, **kwargs):
            lead = None
            new_args = []
            for a in args:
                if torch.is_tensor(a) and a.dim() > n:
                    lead = a.shape[:-(n - 1)]
                    a = a.reshape(-1, *a.shape[-(n - 1):])
                elif torch.is_tensor(a) and 0 < a.dim() < n:
                    lead = () if lead is None else lead
                    a = a.reshape(*([1] * (n - a.dim())), *a.shape)
                new_args.append(a)
            out = fn(*new_args, **kwargs)
            if lead is None:
                return out

            def restore(o):
                if not torch.is_tensor(o):
                    return o
                if lead == ():
                    return o.squeeze(0)
                return o.reshape(*lead, *o.shape[1:])

            if isinstance(out, tuple):
                return tuple(restore(o) for o in out)
            return restore(out)
        return wrapped
    return deco
