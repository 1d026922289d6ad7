"""bevy_b200 -- H100-native per-frame visibility pipeline (propagate -> cull -> cluster).

The product is ``libb200vis.so`` (CUDA kernels for sm_90a behind the C ABI of
``include/b200vis.h``).  This package is its Python host binding: ctypes
plumbing for tests and benchmarks plus a thin mirror of the reference's three
systems.  It never imports ``oracle`` and has no CPU fallback: creating a
context without a CUDA device raises.
"""
from .abi import (  # noqa: F401
    B200VisError, CameraDesc, ColumnSinks, ResultSink, Context, ClusterConfig, ClusterFeedback, ClusterView, FrameStats, View,
    abi_version, host_cluster_view_setup, host_compute_frustum, host_default_cluster_config,
    host_perspective, host_plan_summary, host_z_slice_thresholds, load_library, plan_row_order,
    NO_PARENT, DETACHED, F_INHERITED_VISIBLE, F_HAS_AABB, F_HAS_SPHERE, F_NO_FRUSTUM_CULLING,
    F_HAS_VIS_RANGE, F_NO_CPU_CULLING, F_SPHERE_FROM_GT, VIEW_ACTIVE, VIEW_NO_CPU_CULLING,
    STAGE_PROPAGATE, STAGE_CULL, STAGE_CLUSTER_ASSIGN, STAGE_CLUSTER_LISTS, STAGE_CLUSTER, STAGE_ALL,
)
from .plugin import VisibilityPipeline  # noqa: F401
