"""Packaging of tf_yarn_b200 (reference: setup.py:45-70 -- version, console script).

The native libraries are built in-tree by ``tf_yarn_b200.ops.build`` (``python __graft_entry__.py``);
they are plain C-ABI shared objects loaded with ctypes, so no torch C++ extension machinery is needed.
"""
from setuptools import find_packages, setup

setup(
    name="tf_yarn_b200",
    version="0.2.0",
    description="H100-native distributed-training launcher with the capabilities of criteo/tf-yarn",
    packages=find_packages(include=["tf_yarn_b200", "tf_yarn_b200.*"]),
    package_data={"tf_yarn_b200": ["default.log.conf", "ops/csrc/*", "kv/*.cpp", "examples/*.sh"]},
    python_requires=">=3.10",
    install_requires=["torch", "cloudpickle", "numpy"],
    extras_require={"tensorboard": ["tensorboard"], "parquet": ["pyarrow"], "mlflow": ["mlflow"]},
    entry_points={"console_scripts": ["check_b200_env = tf_yarn_b200.bin.check_env:main",
                                      "check_hadoop_env = tf_yarn_b200.bin.check_hadoop_env:main"]},
)
