"""TEST / BENCH INFRASTRUCTURE ONLY — builds the REFERENCE's own `raymarch_cuda` extension (extensions/ngp_raymarch, setup.py:4-34) for sm_90a, unmodified, from
the reference checkout named by XRB_REF_EXT, into oracle/_ref/cuda/ (git-ignored). Same sources, include dirs and nvcc flags as the reference's setup.py; only
the arch is added. Used by bench.py's `reference_gpu` leg (BASELINE.md B4: the reference's kernels timed on the same GPU next to ours) and by
tests/test_gpu_vs_ref_cuda.py. Nothing in xrnerf_b200/ imports it.

python oracle/build_ref_cuda.py            # ~5 min on 8 cores, once; a no-op when the module is already there or the reference is absent"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get('XRB_REF_EXT', '/root/reference/extensions/ngp_raymarch')
OUT = os.path.join(HERE, '_ref', 'cuda')
NAME = 'raymarch_cuda_ref'
SRCS = ['pybind_api', 'generate_grid_samples_nerf_nonuniform', 'mark_untrained_density_grid', 'splat_grid_samples_nerf_max_nearest_neighbor', 'ema_grid_samples_nerf',
        'update_bitfield', 'ray_sampler', 'compacted_coord', 'calc_rgb']


def module_path():
    p = os.path.join(OUT, NAME + '.so')
    return p if os.path.exists(p) else None


def build(verbose=False):
    if module_path():
        return module_path()
    if not os.path.isdir(os.path.join(REF, 'src')):
        return None
    os.makedirs(OUT, exist_ok=True)
    os.environ['TORCH_CUDA_ARCH_LIST'] = '9.0a'
    os.environ.setdefault('MAX_JOBS', str(os.cpu_count() or 4))
    from torch.utils.cpp_extension import load
    load(name=NAME, sources=[os.path.join(REF, 'src', s + '.cu') for s in SRCS],
         extra_include_paths=[os.path.join(REF, 'include'), os.path.join(REF, 'include', 'op_include', 'eigen'), os.path.join(REF, 'include', 'op_include', 'pcg32')],
         extra_cuda_cflags=['--extended-lambda', '--expt-relaxed-constexpr'], build_directory=OUT, verbose=verbose, is_python_module=False)
    for f in os.listdir(OUT):   # keep the module only
        if not f.endswith('.so'):
            os.remove(os.path.join(OUT, f))
    return module_path()


def load_module():
    """import the prebuilt module (no compiler run, no reference checkout needed)"""
    p = module_path()
    if p is None:
        return None
    import importlib.util
    import torch  # noqa: F401  (libtorch must be loaded first)
    spec = importlib.util.spec_from_file_location(NAME, p)
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


if __name__ == '__main__':
    print(build(verbose='-v' in sys.argv))
