"""
Packaging for the H100-native gossip-SGD framework.

    pip install -e . --no-build-isolation          # builds the sm_90a extension in-tree first

The CUDA extension is NOT a setuptools ``Extension``: it is compiled by
``stochastic_gradient_push_b200/ops/build.py`` (nvcc for the kernels, g++ for the torch
bindings, one ``_C*.so`` next to the package) so that the same artefact serves editable
installs, the test-suite and ``gpurun`` snapshots.  ``build_py`` triggers that build unless
``SGP_B200_SKIP_NATIVE_BUILD=1`` (CPU-only hosts without nvcc can still install the Python side:
every op falls back to its PyTorch composition off-GPU).
"""
import os
import sys

from setuptools import find_packages, setup
from setuptools.command.build_py import build_py


class build_py_with_native(build_py):

    def run(self):
        if os.environ.get('SGP_B200_SKIP_NATIVE_BUILD', '0') == '0':
            sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
            try:
                from stochastic_gradient_push_b200.ops import build as native_build
                print('built', native_build.build())
            except Exception as e:          # no nvcc / no torch headers: Python-only install
                print('WARNING: native extension not built (%s)' % e)
        super().run()


if __name__ == '__main__':
    if sys.version_info < (3, 9):
        sys.exit('Python >= 3.9 is required.')
    here = os.path.dirname(os.path.abspath(__file__))
    with open(os.path.join(here, 'README.md'), encoding='utf8') as f:
        readme = f.read()
    with open(os.path.join(here, 'requirements.txt')) as f:
        reqs = [line.strip() for line in f if line.strip() and not line.startswith('#')]
    setup(
        name='stochastic_gradient_push_b200',
        version='0.1.0',
        description='Gossip-based decentralised data-parallel training (SGP / OSGP / D-PSGD / AD-PSGD) '
                    'with hand-written sm_90a kernels over NVLink peer memory.',
        long_description=readme,
        long_description_content_type='text/markdown',
        python_requires='>=3.9',
        # `gossip` and `experiment_utils` are drop-in aliases of the reference's package names
        packages=find_packages(include=['stochastic_gradient_push_b200*', 'gossip*', 'experiment_utils*',
                                        'visualization*']),
        package_data={'stochastic_gradient_push_b200': ['_C*.so', 'ops/csrc/*']},
        install_requires=reqs,
        extras_require={'parse': ['pandas', 'matplotlib']},
        scripts=['gossip_sgd.py', 'gossip_sgd_adpsgd.py'],
        cmdclass={'build_py': build_py_with_native},
        keywords=['deep learning', 'pytorch', 'decentralized optimization', 'gossip', 'CUDA', 'Hopper'],
        classifiers=['Programming Language :: Python :: 3', 'Environment :: GPU :: NVIDIA CUDA',
                     'Topic :: Scientific/Engineering :: Artificial Intelligence'],
    )
