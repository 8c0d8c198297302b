"""Generate tests/golden/ref_cuda_select.npz: what the reference's own Quantile_T and Isotone_T (thrust::sort, then fixed indices:
ppq/csrc/cuda/sort.cu:6-73) return for inputs where the order of a sort is delicate -- NaNs of both signs and several payloads, +-inf,
runs of +-0 in different input orders, subnormals, n = 1, 2, 3, ranks where n*q is exactly k + 0.5, and n = 2^24 + 1, 2^24 + 3, where
(float)n rounds.  It pins the oracle's reference semantics (oracle.select_t(..., 'reference')) in tests/test_cpu_select_oracle.py.

Needs a CUDA device and the reference's extension built by oracle/build_ref.py (oracle/_ref/PPQ_Cuda_Impls_ref.so):

    python tests/golden/make_ref_select.py [out_dir]          # default: tests/golden

Inputs come from numpy's legacy RandomState and fixed bit patterns (`cases()`), so the CPU test rebuilds them; the two large
inputs are stored as their recipe, not as data.
"""
import importlib.util
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))

NAN_BITS = (0x7FC00000, 0x7F800001, 0x7FFFFFFF, 0x7FA00000, 0xFFC00000, 0xFF800001, 0xFFFFFFFF, 0xFFA00000)
SUBNORMALS = (0x00000001, 0x00000002, 0x007FFFFF, 0x80000001, 0x807FFFFF, 0x00400000)


def u32(bits):
    return np.asarray(bits, dtype=np.uint32).view(np.float32)


def sweep(n):
    """q values whose upper rank rn(n q) visits every index, plus the ends."""
    return [float(np.float32(k) / np.float32(n)) for k in range(n)] + [0.0, 1.0, 0.9999]


def big(n, seed):
    """The large inputs: post-ReLU randn whose zeros carry a random sign, so that the ranks near n/2 select a zero."""
    r = np.random.RandomState(seed)
    x = np.maximum(r.standard_normal(n).astype(np.float32), np.float32(0))
    neg = (x == 0) & (r.rand(n) < 0.5)
    x[neg] = np.float32(-0.0)
    return x


BIG = ((1 << 24) + 1, 11, (0.9999, 0.75, 0.5, 0.25)), ((1 << 24) + 3, 12, (0.9999, 0.6, 0.5, 0.4))


def cases():
    """[(name, x, qs)] of the small inputs."""
    r = np.random.RandomState(2024)
    out = []
    nans = np.concatenate([u32(NAN_BITS), np.float32([np.inf, -np.inf, 1.0, -1.0, 0.0, -0.0])])
    for k in range(3):
        x = nans[r.permutation(nans.size)]
        out.append((f'nan_payloads_{k}', x, sweep(x.size)))
    for k, pattern in enumerate(('--++-', '+-+-+-', '++++--', '-+', '+-', '-0+-0+', '---+')):
        x = np.float32([-0.0 if c == '-' else 0.0 if c == '+' else -1.5 for c in pattern] + [2.0, -3.0])
        out.append((f'zeros_{k}_{pattern}', x, sweep(x.size)))
    for k in range(4):
        x = np.float32(np.where(r.rand(40) < 0.5, -0.0, 0.0))
        x[r.randint(40, size=6)] = r.standard_normal(6).astype(np.float32)
        out.append((f'zero_runs_{k}', x, sweep(x.size)))
    x = np.concatenate([u32(SUBNORMALS), np.float32([0.0, -0.0, 1e-38, -1e-38, -0.0])])
    out.append(('subnormals', x[r.permutation(x.size)], sweep(x.size)))
    for n in (1, 2, 3):
        for k in range(3):
            x = r.choice(np.float32([0.0, -0.0, 1.0, -1.0, np.inf, np.nan]), n).astype(np.float32)
            out.append((f'n{n}_{k}', x, sweep(n) + [0.25, 0.75, 0.5]))
    # n q = k + 0.5 exactly: rn rounds to the even index
    for n, qs in ((4, (0.125, 0.375, 0.625, 0.875)), (8, (0.0625, 0.1875, 0.3125, 0.5625, 0.9375)), (2, (0.25, 0.75))):
        x = r.permutation(np.float32(np.arange(n) - n / 2)).astype(np.float32)
        x[0] = -0.0
        out.append((f'half_ranks_n{n}', x, list(qs)))
    x = r.standard_normal(4099).astype(np.float32)
    x[r.randint(4099, size=300)] = -0.0
    x[r.randint(4099, size=300)] = 0.0
    x[r.randint(4099, size=5)] = u32(NAN_BITS[:5])
    out.append(('mixed_4099', x, [0.9999, 0.99, 0.6, 0.55, 0.5, 0.45, 0.4, 0.0, 1.0]))
    return out


def main(out_dir):
    import torch
    spec = importlib.util.spec_from_file_location('PPQ_Cuda_Impls_ref', os.path.join(ROOT, 'oracle', '_ref', 'PPQ_Cuda_Impls_ref.so'))
    ref = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ref)

    def bits(t):
        return [int(v) for v in t.cpu().numpy().view(np.uint32)]

    small, large = [], []
    for name, x, qs in cases():
        xd = torch.from_numpy(x).cuda()
        small.append({'name': name, 'x': bits(xd), 'q': qs, 'quantile': [bits(ref.Quantile_T(xd, q)) for q in qs],
                      'isotone': bits(ref.Isotone_T(xd))})
    for n, seed, qs in BIG:
        xd = torch.from_numpy(big(n, seed)).cuda()
        large.append({'n': n, 'seed': seed, 'q': list(qs), 'quantile': [bits(ref.Quantile_T(xd, q)) for q in qs],
                      'isotone': bits(ref.Isotone_T(xd))})
    os.makedirs(out_dir, exist_ok=True)
    path = os.path.join(out_dir, 'ref_cuda_select.npz')
    np.savez_compressed(path, cases=np.frombuffer(json.dumps({'small': small, 'large': large}).encode(), np.uint8),
                        device=np.frombuffer(torch.cuda.get_device_name(0).encode(), np.uint8))
    print('wrote', path, len(small), 'small and', len(large), 'large cases')


if __name__ == '__main__':
    main(sys.argv[1] if len(sys.argv) > 1 else HERE)
