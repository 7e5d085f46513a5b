"""ctypes binding of libgangpack.so (include/gangpack.h) -- the only compute path of this package.

There is deliberately no CPU fallback here: if the shared library is missing or no sm_90 device is
usable, loading / context creation raises.
"""
from __future__ import annotations

import ctypes as C
import glob
import os
import shutil
import subprocess

import numpy as np

_PKG = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_PKG)
LIB_PATH = os.environ.get("GANGPACK_LIB") or os.path.join(_PKG, "libgangpack.so")   # GANGPACK_LIB: experimental builds

NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
              "-shared", "-Xcompiler", "-fPIC"]

TIGHTLY_PACK = 0
DISTRIBUTE_EVENLY = 1
MINIMAL_FRAGMENTATION = 2   # GP_MODE_INDEPENDENT only
MODE_INDEPENDENT = 0
MODE_FIFO_REFERENCE = 1
MODE_FIFO_EXACT = 2

STATUS_NAMES = {0: "GP_OK", 1: "GP_ERR_INVALID", 2: "GP_ERR_CUDA", 3: "GP_ERR_NO_DEVICE", 4: "GP_ERR_NO_SNAPSHOT",
                5: "GP_ERR_CAPACITY", 6: "GP_ERR_UNREPRESENTABLE"}

# every symbol include/gangpack.h declares (tests assert the .so exports exactly these)
EXPORTS = ["gp_abi_version", "gp_create", "gp_destroy", "gp_last_error", "gp_backend", "gp_alloc_pinned",
           "gp_free_pinned", "gp_register_host", "gp_unregister_host", "gp_set_snapshot", "gp_get_snapshot", "gp_pack_batch", "gp_pack_batch_wire", "gp_pack_one", "gp_set_schedulable", "gp_pack_batch_zones", "gp_pack_fifo_zones", "gp_pack_fifo_az_aware", "gp_pack_batch_az_aware", "gp_reserve_placements", "gp_apply_usage_delta",
           "gp_set_snapshot_device", "gp_pack_batch_device", "gp_stream", "gp_synchronize", "gp_last_stats",
           "gp_potential_nodes", "gp_build_availability", "gp_build_reschedule_availability", "gp_prepare_cluster", "gp_prepare_cluster_zones",
           "gp_reschedule_executors", "gp_reschedule_from_reservations", "gp_packing_efficiency", "gp_exceeds_cluster_capacity",
           "gp_reconcile_find_nodes", "gp_match_node_affinity", "gp_exceeds_cluster_capacity_affinity",
           "gp_node_overhead", "gp_overhead_table_reset", "gp_overhead_table_update", "gp_overhead_table_query",
           "gp_reservation_table_reset", "gp_reservation_table_update", "gp_prepare_cluster_groups_resident",
           "gp_prepare_cluster_zones_groups_resident", "gp_reschedule_from_reservations_resident",
           "gp_reconcile_find_nodes_resident", "gp_exceeds_cluster_capacity_resident",
           "gp_exceeds_cluster_capacity_affinity_resident", "gp_label_table_reset", "gp_label_table_update",
           "gp_match_node_affinity_resident", "gp_exceeds_cluster_capacity_affinity_label_table",
           "gp_node_table_reset", "gp_node_table_update", "gp_prepare_cluster_groups_node_table",
           "gp_prepare_cluster_zones_groups_node_table", "gp_reschedule_from_reservations_node_table",
           "gp_reconcile_find_nodes_node_table", "gp_exceeds_cluster_capacity_node_table",
           "gp_exceeds_cluster_capacity_affinity_node_table",
           "gp_driver_table_reset", "gp_driver_table_update", "gp_pack_fifo_driver_table",
           "gp_pack_fifo_zones_groups_driver_table", "gp_exceeds_cluster_capacity_driver_table",
           "gp_pack_fifo_zones_groups", "gp_prepare_cluster_zones_groups",
           "gp_prepare_cluster_groups", "gp_packing_efficiency_groups", "gp_placement_metrics", "gp_placement_metrics_device",
           "gp_multi_create", "gp_multi_destroy", "gp_multi_last_error", "gp_multi_size", "gp_multi_ctx",
           "gp_multi_set_snapshot", "gp_multi_pack_batch", "gp_multi_get_snapshot", "gp_multi_group_owner"]


class GangpackError(RuntimeError):
    def __init__(self, status: int, message: str):
        super().__init__(f"{STATUS_NAMES.get(status, status)}: {message}")
        self.status = status


def _nvcc() -> str:
    for cand in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found; cannot build libgangpack.so")


def build(force: bool = False, verbose: bool = False, out: str | None = None, defines=()) -> str:
    """Compile csrc/*.cu for sm_90a into k8s-spark-scheduler_b200/libgangpack.so (in-tree), or into `out` with extra
    preprocessor `defines` (diagnostic builds such as GP_DECIDE_TIMELINE; never the in-tree library)."""
    path = out or LIB_PATH
    csrc = os.path.join(_PKG, "csrc")
    units = sorted(glob.glob(os.path.join(csrc, "*.cu")))
    inputs = units + glob.glob(os.path.join(csrc, "*.cuh")) + [os.path.join(_ROOT, "include", "gangpack.h")]
    stale = force or not os.path.exists(path) or any(
        os.path.getmtime(s) > os.path.getmtime(path) for s in inputs)
    if stale:
        cmd = [_nvcc()] + NVCC_FLAGS + [f"-D{d}" for d in defines] + [
            "-I", os.path.join(_ROOT, "include"), "-o", path] + units
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        subprocess.check_call(cmd)
    return path


class gp_config(C.Structure):
    _fields_ = [("device", C.c_int32), ("flags", C.c_int32), ("reserved", C.c_int32 * 6)]


CFG_ASYNC_SNAPSHOT = 1


class gp_nodes(C.Structure):
    _fields_ = [("n_nodes", C.c_int32), ("avail_cpu_milli", C.c_void_p), ("avail_mem_bytes", C.c_void_p),
                ("avail_gpu", C.c_void_p), ("n_groups", C.c_int32), ("exec_off", C.c_void_p),
                ("exec_order", C.c_void_p), ("drv_off", C.c_void_p), ("drv_order", C.c_void_p)]


class gp_apps(C.Structure):
    _fields_ = [("n_apps", C.c_int32), ("drv_cpu_milli", C.c_void_p), ("drv_mem_bytes", C.c_void_p),
                ("drv_gpu", C.c_void_p), ("exe_cpu_milli", C.c_void_p), ("exe_mem_bytes", C.c_void_p),
                ("exe_gpu", C.c_void_p), ("exe_count", C.c_void_p), ("group", C.c_void_p),
                ("skip_if_no_fit", C.c_void_p), ("exec_out_off", C.c_void_p)]


class gp_apps_wire(C.Structure):
    _fields_ = [("n_apps", C.c_int32), ("quantity_bits", C.c_int32), ("mem_shift", C.c_int32), ("reserved", C.c_int32),
                ("drv_cpu", C.c_void_p), ("drv_mem", C.c_void_p), ("drv_gpu", C.c_void_p),
                ("exe_cpu", C.c_void_p), ("exe_mem", C.c_void_p), ("exe_gpu", C.c_void_p),
                ("exe_count", C.c_void_p), ("group", C.c_void_p), ("skip_if_no_fit", C.c_void_p), ("exec_out_off", C.c_void_p)]


class gp_results_wire(C.Structure):
    _fields_ = [("driver_node", C.c_void_p), ("executor_nodes", C.c_void_p), ("executor_nodes_cap", C.c_int64),
                ("node_bits", C.c_int32), ("reserved", C.c_int32)]


class gp_zone_results(C.Structure):
    _fields_ = [("zone", C.c_void_p), ("driver_node", C.c_void_p), ("executor_nodes", C.c_void_p), ("executor_nodes_cap", C.c_int64),
                ("avg_efficiency", C.c_void_p)]


class gp_az_orders(C.Structure):
    _fields_ = [("n_zones", C.c_int32), ("n_exec", C.c_int32), ("exec_order", C.c_void_p), ("n_drv", C.c_int32),
                ("drv_order", C.c_void_p)]


class gp_instance_groups(C.Structure):
    _fields_ = [("n_instance_groups", C.c_int32), ("group_off", C.c_void_p), ("n_zones", C.c_void_p), ("exec_off", C.c_void_p),
                ("exec_order", C.c_void_p), ("drv_off", C.c_void_p), ("drv_order", C.c_void_p)]


class gp_reservation_table(C.Structure):
    _fields_ = [("rows_cap", C.c_int64), ("app", C.c_void_p), ("slot", C.c_void_p), ("node", C.c_void_p), ("cpu_milli", C.c_void_p),
                ("mem_bytes", C.c_void_p), ("gpu", C.c_void_p), ("n_rows", C.c_int64)]


class gp_results(C.Structure):
    _fields_ = [("driver_node", C.c_void_p), ("executor_nodes", C.c_void_p), ("executor_nodes_cap", C.c_int64)]


class gp_sort_input(C.Structure):
    _fields_ = [("n_nodes", C.c_int32), ("avail_cpu_milli", C.c_void_p), ("avail_mem_bytes", C.c_void_p),
                ("n_zones", C.c_int32), ("zone_id", C.c_void_p), ("name_rank", C.c_void_p),
                ("is_driver_candidate", C.c_void_p), ("unschedulable", C.c_void_p), ("ready", C.c_void_p),
                ("driver_label_rank", C.c_void_p), ("executor_label_rank", C.c_void_p),
                ("avail_gpu", C.c_void_p), ("undefined_ties", C.c_void_p)]


class gp_usage_input(C.Structure):
    _fields_ = [("n_nodes", C.c_int32), ("alloc_cpu_milli", C.c_void_p), ("alloc_mem_bytes", C.c_void_p), ("alloc_gpu", C.c_void_p),
                ("overhead_cpu_milli", C.c_void_p), ("overhead_mem_bytes", C.c_void_p), ("overhead_gpu", C.c_void_p),
                ("n_reservations", C.c_int64), ("res_node", C.c_void_p), ("res_cpu_milli", C.c_void_p),
                ("res_mem_bytes", C.c_void_p), ("res_gpu", C.c_void_p)]


LAYOUT_SINGLE_AZ = 0
LAYOUT_AZ_AWARE = 1


class gp_zone_layout(C.Structure):
    _fields_ = [("kind", C.c_int32), ("n_zones", C.c_int32), ("n_groups", C.c_int32), ("n_driver", C.c_int32),
                ("n_executor", C.c_int32), ("reserved", C.c_int32), ("zone_of_group", C.c_void_p), ("exec_off", C.c_void_p),
                ("exec_order", C.c_void_p), ("drv_off", C.c_void_p), ("drv_order", C.c_void_p)]


class gp_instance_group_layout(C.Structure):
    _fields_ = [("kind", C.c_int32), ("n_groups", C.c_int32), ("n_driver", C.c_int32), ("n_executor", C.c_int32)] + \
        [(k, C.c_void_p) for k in ("group_off", "n_zones", "exec_off", "exec_order", "drv_off", "drv_order", "group_exec_off",
                                   "group_exec_order", "group_drv_off", "group_drv_order", "zone_of_group", "undefined_ties")]


class gp_instance_group_orders(C.Structure):
    _fields_ = [("n_driver", C.c_int32), ("n_executor", C.c_int32)] + \
        [(k, C.c_void_p) for k in ("exec_off", "exec_order", "drv_off", "drv_order", "undefined_ties")]


class gp_reschedule(C.Structure):
    _fields_ = [("n_execs", C.c_int32), ("exe_cpu_milli", C.c_void_p), ("exe_mem_bytes", C.c_void_p), ("exe_gpu", C.c_void_p),
                ("group", C.c_void_p), ("min_frag", C.c_int32), ("reserved_cpu_milli", C.c_void_p),
                ("reserved_mem_bytes", C.c_void_p), ("reserved_gpu", C.c_void_p), ("host_off", C.c_void_p),
                ("host_nodes", C.c_void_p)]


class gp_reschedule_scope(C.Structure):
    _fields_ = [("keep_topology_zone", C.c_int32), ("reserved", C.c_int32), ("topology_zone", C.c_void_p)]


# gp_binpacker: the `binpack:` config values (internal/binpacker/binpack.go:21-24, 43-49)
BP_TIGHTLY_PACK = 0
BP_DISTRIBUTE_EVENLY = 1
BP_AZ_AWARE_TIGHTLY_PACK = 2
BP_SINGLE_AZ_TIGHTLY_PACK = 3
BP_SINGLE_AZ_MINIMAL_FRAGMENTATION = 4
BINPACKERS = {"tightly-pack": BP_TIGHTLY_PACK, "distribute-evenly": BP_DISTRIBUTE_EVENLY,
              "az-aware-tightly-pack": BP_AZ_AWARE_TIGHTLY_PACK, "single-az-tightly-pack": BP_SINGLE_AZ_TIGHTLY_PACK,
              "single-az-minimal-fragmentation": BP_SINGLE_AZ_MINIMAL_FRAGMENTATION}


class gp_capacity_nodes(C.Structure):
    _fields_ = [("n_nodes", C.c_int32), ("alloc_cpu_milli", C.c_void_p), ("alloc_mem_bytes", C.c_void_p), ("alloc_gpu", C.c_void_p),
                ("overhead_cpu_milli", C.c_void_p), ("overhead_mem_bytes", C.c_void_p), ("overhead_gpu", C.c_void_p),
                ("n_zones", C.c_int32), ("zone_id", C.c_void_p), ("n_groups", C.c_int32), ("node_group", C.c_void_p)]


class gp_node_labels(C.Structure):
    _fields_ = [("n_nodes", C.c_int32), ("n_keys", C.c_int32), ("n_values", C.c_int32), ("reserved", C.c_int32),
                ("label_off", C.c_void_p), ("label_key", C.c_void_p), ("label_val", C.c_void_p), ("label_int_ok", C.c_void_p),
                ("label_int", C.c_void_p)]


class gp_node_affinities(C.Structure):
    _fields_ = [("n_aff", C.c_int32), ("reserved", C.c_int32), ("sel_off", C.c_void_p), ("sel_key", C.c_void_p),
                ("sel_val", C.c_void_p), ("has_required", C.c_void_p), ("term_off", C.c_void_p), ("term_req_off", C.c_void_p),
                ("term_parse_error", C.c_void_p), ("req_op", C.c_void_p), ("req_key", C.c_void_p), ("req_int", C.c_void_p),
                ("req_val_off", C.c_void_p), ("req_val", C.c_void_p)]


class gp_affinity_match(C.Structure):
    _fields_ = [("member", C.c_void_p), ("n_match", C.c_void_p), ("n_error", C.c_void_p)]


class gp_reconcile_nodes(C.Structure):
    _fields_ = [("n_groups", C.c_int32), ("reserved", C.c_int32), ("node_group", C.c_void_p), ("creation", C.c_void_p),
                ("unschedulable", C.c_void_p), ("ready", C.c_void_p)]


class gp_reconcile_results(C.Structure):
    _fields_ = [("placed", C.c_void_p), ("executor_nodes", C.c_void_p), ("executor_nodes_cap", C.c_int64),
                ("avail_cpu_milli", C.c_void_p), ("avail_mem_bytes", C.c_void_p), ("avail_gpu", C.c_void_p)]


class gp_overhead_pods(C.Structure):
    _fields_ = [("n_pods", C.c_int64), ("n_node_ids", C.c_int32), ("n_app_keys", C.c_int32), ("n_app_ids", C.c_int32),
                ("n_names", C.c_int32), ("node_id", C.c_void_p), ("req_cpu_milli", C.c_void_p), ("req_mem_bytes", C.c_void_p),
                ("req_gpu", C.c_void_p), ("listed", C.c_void_p), ("app_key", C.c_void_p), ("app_id", C.c_void_p),
                ("name_id", C.c_void_p), ("is_executor", C.c_void_p), ("spark_scheduler", C.c_void_p)]


class gp_overhead_reservations(C.Structure):
    _fields_ = [("n_rr", C.c_int32), ("n_soft", C.c_int32), ("rr_app_key", C.c_void_p), ("rr_pod_off", C.c_void_p),
                ("rr_pod_name", C.c_void_p), ("soft_app_id", C.c_void_p), ("soft_pod_off", C.c_void_p), ("soft_pod_name", C.c_void_p)]


class gp_overhead_out(C.Structure):
    _fields_ = [("overhead_cpu_milli", C.c_void_p), ("overhead_mem_bytes", C.c_void_p), ("overhead_gpu", C.c_void_p),
                ("nonsched_cpu_milli", C.c_void_p), ("nonsched_mem_bytes", C.c_void_p), ("nonsched_gpu", C.c_void_p),
                ("has_reservation", C.c_void_p), ("n_warned", C.c_void_p)]


class gp_overhead_table_size(C.Structure):
    _fields_ = [("n_slots", C.c_int64), ("n_node_ids", C.c_int32), ("n_app_keys", C.c_int32), ("n_app_ids", C.c_int32),
                ("n_names", C.c_int32)]


class gp_overhead_delta(C.Structure):
    _fields_ = [("n_write", C.c_int64), ("slot", C.c_void_p), ("node_id", C.c_void_p), ("req_cpu_milli", C.c_void_p),
                ("req_mem_bytes", C.c_void_p), ("req_gpu", C.c_void_p), ("listed", C.c_void_p), ("app_key", C.c_void_p),
                ("app_id", C.c_void_p), ("name_id", C.c_void_p), ("is_executor", C.c_void_p), ("spark_scheduler", C.c_void_p),
                ("n_rr", C.c_int32), ("rr_app_key", C.c_void_p), ("rr_exists", C.c_void_p), ("n_member", C.c_int64),
                ("member_kind", C.c_void_p), ("member_app", C.c_void_p), ("member_name", C.c_void_p), ("member_present", C.c_void_p)]


class gp_reservation_table_size(C.Structure):
    _fields_ = [("n_slots", C.c_int64), ("n_node_ids", C.c_int32)]


class gp_reservation_delta(C.Structure):
    _fields_ = [("n_write", C.c_int64), ("slot", C.c_void_p), ("node_id", C.c_void_p), ("cpu_milli", C.c_void_p),
                ("mem_bytes", C.c_void_p), ("gpu", C.c_void_p)]


class gp_resident_usage(C.Structure):
    _fields_ = [("n_nodes", C.c_int32), ("node_id", C.c_void_p), ("alloc_cpu_milli", C.c_void_p), ("alloc_mem_bytes", C.c_void_p),
                ("alloc_gpu", C.c_void_p), ("overhead_node_id", C.c_void_p), ("overhead_cpu_milli", C.c_void_p),
                ("overhead_mem_bytes", C.c_void_p), ("overhead_gpu", C.c_void_p)]


class gp_label_table_size(C.Structure):
    _fields_ = [("n_node_ids", C.c_int32), ("max_labels", C.c_int32), ("n_keys", C.c_int32), ("n_values", C.c_int32)]


class gp_label_delta(C.Structure):
    _fields_ = [("n_rows", C.c_int32), ("n_values", C.c_int32), ("row_node", C.c_void_p), ("row_off", C.c_void_p),
                ("label_key", C.c_void_p), ("label_val", C.c_void_p), ("value_id", C.c_void_p), ("value_int_ok", C.c_void_p),
                ("value_int", C.c_void_p)]


class gp_resident_labels(C.Structure):
    _fields_ = [("n_nodes", C.c_int32), ("reserved", C.c_int32), ("node_id", C.c_void_p)]


class gp_node_table_size(C.Structure):
    _fields_ = [("n_node_ids", C.c_int32), ("reserved", C.c_int32)]


class gp_node_delta(C.Structure):
    _fields_ = [("n_write", C.c_int32), ("reserved", C.c_int32), ("node_id", C.c_void_p), ("present", C.c_void_p),
                ("alloc_cpu_milli", C.c_void_p), ("alloc_mem_bytes", C.c_void_p), ("alloc_gpu", C.c_void_p),
                ("unschedulable", C.c_void_p), ("ready", C.c_void_p), ("name_key", C.c_void_p), ("creation", C.c_void_p)]


class gp_node_table_nodes(C.Structure):
    _fields_ = [("n_nodes", C.c_int32), ("reserved", C.c_int32), ("node_table_id", C.c_void_p), ("reservation_id", C.c_void_p),
                ("overhead_node_id", C.c_void_p), ("is_driver_candidate", C.c_void_p), ("zone_key", C.c_int32), ("n_zones", C.c_int32),
                ("zone_value", C.c_void_p), ("zone_missing", C.c_int32), ("instance_group_key", C.c_int32),
                ("instance_group_value", C.c_void_p), ("driver_rank_key", C.c_int32), ("n_driver_rank_values", C.c_int32),
                ("driver_rank_value", C.c_void_p), ("executor_rank_key", C.c_int32), ("n_executor_rank_values", C.c_int32),
                ("executor_rank_value", C.c_void_p), ("undefined_ties", C.c_void_p), ("zone_id_out", C.c_void_p),
                ("instance_group_out", C.c_void_p)]


class gp_driver_table_size(C.Structure):
    _fields_ = [("n_slots", C.c_int32), ("n_groups", C.c_int32), ("n_schedulers", C.c_int32), ("reserved", C.c_int32)]


class gp_driver_delta(C.Structure):
    _fields_ = [("n_write", C.c_int32), ("reserved", C.c_int32), ("slot", C.c_void_p), ("present", C.c_void_p),
                ("creation", C.c_void_p), ("scheduler", C.c_void_p), ("group", C.c_void_p), ("drv_cpu_milli", C.c_void_p),
                ("drv_mem_bytes", C.c_void_p), ("drv_gpu", C.c_void_p), ("exe_cpu_milli", C.c_void_p), ("exe_mem_bytes", C.c_void_p),
                ("exe_gpu", C.c_void_p), ("min_executor_count", C.c_void_p), ("exact", C.c_void_p), ("affinity", C.c_void_p)]


class gp_driver_queue(C.Structure):
    _fields_ = [("requesting_slot", C.c_int32), ("scheduler", C.c_int32), ("predicate_group", C.c_int32), ("queue_cap", C.c_int32),
                ("snapshot_group", C.c_void_p), ("enforce_after_ns", C.c_void_p), ("now_unix_nano", C.c_int64),
                ("queue_slot", C.c_void_p), ("exec_out_off", C.c_void_p), ("n_queued", C.c_void_p), ("n_executors", C.c_void_p),
                ("undefined_ties", C.c_void_p)]


class gp_stale_sweep(C.Structure):
    _fields_ = [("scheduler", C.c_int32), ("cap", C.c_int32), ("timeout_ns", C.c_int64), ("now_unix_nano", C.c_int64),
                ("stale_slot", C.c_void_p), ("exceeds", C.c_void_p), ("outcome", C.c_void_p), ("n_stale", C.c_void_p)]


class gp_placement_record(C.Structure):
    _fields_ = [("collocation", C.c_int32), ("distinct_exec_nodes", C.c_int32), ("execs_per_node", C.c_int32), ("n_zones", C.c_int32),
                ("cross_zone_pairs", C.c_int64), ("total_pairs", C.c_int64)]


# numpy view of gp_placement_record[]: collocation -1 = not reported (driver_node < 0), 0 no-collocation,
# 1 driver-collocated-with-all-executors, 2 driver-collocated-with-some-executors
PLACEMENT_DTYPE = np.dtype([(f, np.int32 if t is C.c_int32 else np.int64) for f, t in gp_placement_record._fields_])
COLLOCATION_TAGS = {0: "no-collocation", 1: "driver-collocated-with-all-executors", 2: "driver-collocated-with-some-executors"}


class gp_stats(C.Structure):
    _fields_ = [("nodes_scanned", C.c_int64), ("drivers_tried", C.c_int64), ("kernel_launches", C.c_int64),
                ("pack_kernel_ns", C.c_int64), ("prep_kernel_ns", C.c_int64), ("scan_path_apps", C.c_int64),
                ("scan_path_nodes", C.c_int64), ("reserved", C.c_int64 * 1)]


_lib = None


def load():
    """dlopen libgangpack.so; raises if it has not been built (no silent fallback)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                           "(this package has no CPU fallback)")
    L = C.CDLL(LIB_PATH)
    L.gp_abi_version.restype = C.c_int
    L.gp_create.restype = C.c_int
    L.gp_create.argtypes = [C.POINTER(C.c_void_p), C.POINTER(gp_config)]
    L.gp_destroy.restype = None
    L.gp_destroy.argtypes = [C.c_void_p]
    L.gp_last_error.restype = C.c_char_p
    L.gp_last_error.argtypes = [C.c_void_p]
    L.gp_backend.restype = C.c_int
    L.gp_backend.argtypes = [C.c_void_p]
    L.gp_alloc_pinned.restype = C.c_int
    L.gp_alloc_pinned.argtypes = [C.c_void_p, C.c_size_t, C.POINTER(C.c_void_p)]
    L.gp_free_pinned.restype = C.c_int
    L.gp_free_pinned.argtypes = [C.c_void_p, C.c_void_p]
    L.gp_register_host.restype = C.c_int
    L.gp_register_host.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
    L.gp_unregister_host.restype = C.c_int
    L.gp_unregister_host.argtypes = [C.c_void_p, C.c_void_p]
    L.gp_set_snapshot.restype = C.c_int
    L.gp_set_snapshot.argtypes = [C.c_void_p, C.POINTER(gp_nodes)]
    L.gp_get_snapshot.restype = C.c_int
    L.gp_get_snapshot.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.gp_pack_batch.restype = C.c_int
    L.gp_pack_batch.argtypes = [C.c_void_p, C.POINTER(gp_apps), C.c_int, C.c_int, C.POINTER(gp_results)]
    L.gp_pack_batch_wire.restype = C.c_int
    L.gp_pack_batch_wire.argtypes = [C.c_void_p, C.POINTER(gp_apps_wire), C.c_int, C.c_int, C.POINTER(gp_results_wire)]
    L.gp_set_schedulable.restype = C.c_int
    L.gp_set_schedulable.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.gp_pack_batch_zones.restype = C.c_int
    L.gp_pack_batch_zones.argtypes = [C.c_void_p, C.POINTER(gp_apps), C.c_int, C.POINTER(gp_zone_results)]
    L.gp_pack_fifo_zones.restype = C.c_int
    L.gp_pack_fifo_zones.argtypes = [C.c_void_p, C.POINTER(gp_apps), C.c_int, C.c_int, C.POINTER(gp_zone_results)]
    L.gp_pack_fifo_az_aware.restype = C.c_int
    L.gp_pack_fifo_az_aware.argtypes = [C.c_void_p, C.POINTER(gp_apps), C.c_int, C.POINTER(gp_az_orders), C.POINTER(gp_zone_results)]
    L.gp_pack_batch_az_aware.restype = C.c_int
    L.gp_pack_batch_az_aware.argtypes = [C.c_void_p, C.POINTER(gp_apps), C.POINTER(gp_az_orders), C.POINTER(gp_zone_results)]
    L.gp_pack_fifo_zones_groups.restype = C.c_int
    L.gp_pack_fifo_zones_groups.argtypes = [C.c_void_p, C.POINTER(gp_apps), C.c_int, C.c_int, C.POINTER(gp_instance_groups),
                                            C.POINTER(gp_zone_results)]
    L.gp_reserve_placements.restype = C.c_int
    L.gp_reserve_placements.argtypes = [C.c_void_p, C.POINTER(gp_apps), C.POINTER(gp_results), C.c_int32, C.POINTER(gp_reservation_table)]
    L.gp_apply_usage_delta.restype = C.c_int
    L.gp_apply_usage_delta.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32]
    L.gp_packing_efficiency.restype = C.c_int
    L.gp_packing_efficiency.argtypes = [C.c_void_p, C.POINTER(gp_apps), C.c_int, C.POINTER(gp_results), C.c_int, C.c_void_p]
    L.gp_packing_efficiency_groups.restype = C.c_int
    L.gp_packing_efficiency_groups.argtypes = [C.c_void_p, C.POINTER(gp_apps), C.c_int, C.POINTER(gp_results), C.c_int, C.c_void_p,
                                               C.c_int32, C.c_void_p]
    L.gp_exceeds_cluster_capacity.restype = C.c_int
    L.gp_placement_metrics.restype = C.c_int
    L.gp_placement_metrics.argtypes = [C.c_void_p, C.POINTER(gp_apps), C.POINTER(gp_results), C.c_int32, C.c_void_p, C.c_int32,
                                       C.c_void_p, C.c_int32, C.c_void_p]
    L.gp_placement_metrics_device.restype = C.c_int
    L.gp_placement_metrics_device.argtypes = [C.c_void_p, C.POINTER(gp_apps), C.POINTER(gp_results), C.c_int32, C.c_void_p,
                                              C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
    L.gp_exceeds_cluster_capacity.argtypes = [C.c_void_p, C.POINTER(gp_capacity_nodes), C.POINTER(gp_apps), C.c_int, C.c_void_p]
    L.gp_reconcile_find_nodes.restype = C.c_int
    L.gp_match_node_affinity.restype = C.c_int
    L.gp_match_node_affinity.argtypes = [C.c_void_p, C.POINTER(gp_node_labels), C.POINTER(gp_node_affinities), C.POINTER(gp_affinity_match)]
    L.gp_exceeds_cluster_capacity_affinity.restype = C.c_int
    L.gp_exceeds_cluster_capacity_affinity.argtypes = [C.c_void_p, C.POINTER(gp_capacity_nodes), C.POINTER(gp_node_labels),
                                                       C.POINTER(gp_node_affinities), C.POINTER(gp_apps), C.c_int, C.c_void_p,
                                                       C.c_void_p]
    L.gp_reconcile_find_nodes.argtypes = [C.c_void_p, C.POINTER(gp_usage_input), C.POINTER(gp_reconcile_nodes), C.POINTER(gp_apps),
                                          C.POINTER(gp_reconcile_results)]
    L.gp_node_overhead.restype = C.c_int
    L.gp_node_overhead.argtypes = [C.c_void_p, C.POINTER(gp_overhead_pods), C.POINTER(gp_overhead_reservations), C.c_int32,
                                   C.c_void_p, C.POINTER(gp_overhead_out)]
    L.gp_overhead_table_reset.restype = C.c_int
    L.gp_overhead_table_reset.argtypes = [C.c_void_p, C.POINTER(gp_overhead_table_size)]
    L.gp_overhead_table_update.restype = C.c_int
    L.gp_overhead_table_update.argtypes = [C.c_void_p, C.POINTER(gp_overhead_delta)]
    L.gp_overhead_table_query.restype = C.c_int
    L.gp_overhead_table_query.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.POINTER(gp_overhead_out)]
    L.gp_reservation_table_reset.restype = C.c_int
    L.gp_reservation_table_reset.argtypes = [C.c_void_p, C.POINTER(gp_reservation_table_size)]
    L.gp_reservation_table_update.restype = C.c_int
    L.gp_reservation_table_update.argtypes = [C.c_void_p, C.POINTER(gp_reservation_delta)]
    L.gp_prepare_cluster_groups_resident.restype = C.c_int
    L.gp_prepare_cluster_groups_resident.argtypes = [C.c_void_p, C.POINTER(gp_resident_usage), C.POINTER(gp_sort_input), C.c_void_p,
                                                     C.c_int32, C.POINTER(gp_instance_group_orders)]
    L.gp_prepare_cluster_zones_groups_resident.restype = C.c_int
    L.gp_prepare_cluster_zones_groups_resident.argtypes = [C.c_void_p, C.POINTER(gp_resident_usage), C.POINTER(gp_sort_input),
                                                           C.c_void_p, C.c_int32, C.POINTER(gp_instance_group_layout)]
    L.gp_reconcile_find_nodes_resident.restype = C.c_int
    L.gp_reconcile_find_nodes_resident.argtypes = [C.c_void_p, C.POINTER(gp_resident_usage), C.POINTER(gp_reconcile_nodes),
                                                   C.POINTER(gp_apps), C.POINTER(gp_reconcile_results)]
    L.gp_exceeds_cluster_capacity_resident.restype = C.c_int
    L.gp_exceeds_cluster_capacity_resident.argtypes = [C.c_void_p, C.POINTER(gp_capacity_nodes), C.c_void_p, C.POINTER(gp_apps), C.c_int,
                                                       C.c_void_p]
    L.gp_exceeds_cluster_capacity_affinity_resident.restype = C.c_int
    L.gp_exceeds_cluster_capacity_affinity_resident.argtypes = [C.c_void_p, C.POINTER(gp_capacity_nodes), C.c_void_p,
                                                                C.POINTER(gp_node_labels), C.POINTER(gp_node_affinities),
                                                                C.POINTER(gp_apps), C.c_int, C.c_void_p, C.c_void_p]
    L.gp_label_table_reset.restype = C.c_int
    L.gp_label_table_reset.argtypes = [C.c_void_p, C.POINTER(gp_label_table_size)]
    L.gp_label_table_update.restype = C.c_int
    L.gp_label_table_update.argtypes = [C.c_void_p, C.POINTER(gp_label_delta)]
    L.gp_match_node_affinity_resident.restype = C.c_int
    L.gp_match_node_affinity_resident.argtypes = [C.c_void_p, C.POINTER(gp_resident_labels), C.POINTER(gp_node_affinities),
                                                  C.POINTER(gp_affinity_match)]
    L.gp_exceeds_cluster_capacity_affinity_label_table.restype = C.c_int
    L.gp_exceeds_cluster_capacity_affinity_label_table.argtypes = [C.c_void_p, C.POINTER(gp_capacity_nodes), C.c_void_p,
                                                                   C.POINTER(gp_resident_labels), C.POINTER(gp_node_affinities),
                                                                   C.POINTER(gp_apps), C.c_int, C.c_void_p, C.c_void_p]
    L.gp_reschedule_from_reservations_resident.restype = C.c_int
    L.gp_reschedule_from_reservations_resident.argtypes = [C.c_void_p, C.POINTER(gp_resident_usage), C.POINTER(gp_sort_input),
                                                           C.POINTER(gp_reschedule_scope), C.POINTER(gp_reschedule), C.c_void_p,
                                                           C.c_void_p]
    L.gp_node_table_reset.restype = C.c_int
    L.gp_node_table_reset.argtypes = [C.c_void_p, C.POINTER(gp_node_table_size)]
    L.gp_node_table_update.restype = C.c_int
    L.gp_node_table_update.argtypes = [C.c_void_p, C.POINTER(gp_node_delta)]
    L.gp_prepare_cluster_groups_node_table.restype = C.c_int
    L.gp_prepare_cluster_groups_node_table.argtypes = [C.c_void_p, C.POINTER(gp_node_table_nodes), C.c_void_p, C.c_int32,
                                                       C.POINTER(gp_instance_group_orders)]
    L.gp_prepare_cluster_zones_groups_node_table.restype = C.c_int
    L.gp_prepare_cluster_zones_groups_node_table.argtypes = [C.c_void_p, C.POINTER(gp_node_table_nodes), C.c_void_p, C.c_int32,
                                                             C.POINTER(gp_instance_group_layout)]
    L.gp_reschedule_from_reservations_node_table.restype = C.c_int
    L.gp_reschedule_from_reservations_node_table.argtypes = [C.c_void_p, C.POINTER(gp_node_table_nodes), C.POINTER(gp_reschedule_scope),
                                                             C.POINTER(gp_reschedule), C.c_void_p, C.c_void_p]
    L.gp_reconcile_find_nodes_node_table.restype = C.c_int
    L.gp_reconcile_find_nodes_node_table.argtypes = [C.c_void_p, C.POINTER(gp_node_table_nodes), C.c_int32, C.c_int32, C.POINTER(gp_apps),
                                                     C.POINTER(gp_reconcile_results)]
    L.gp_exceeds_cluster_capacity_node_table.restype = C.c_int
    L.gp_exceeds_cluster_capacity_node_table.argtypes = [C.c_void_p, C.POINTER(gp_node_table_nodes), C.c_void_p, C.c_int32,
                                                         C.POINTER(gp_apps), C.c_int, C.c_void_p]
    L.gp_exceeds_cluster_capacity_affinity_node_table.restype = C.c_int
    L.gp_exceeds_cluster_capacity_affinity_node_table.argtypes = [C.c_void_p, C.POINTER(gp_node_table_nodes), C.POINTER(gp_node_affinities),
                                                                  C.POINTER(gp_apps), C.c_int, C.c_void_p, C.c_void_p]
    L.gp_pack_one.restype = C.c_int
    L.gp_pack_one.argtypes = [C.c_void_p, C.c_int] + [C.c_int64] * 6 + [C.c_int32, C.POINTER(C.c_int32),
                                                                          C.POINTER(C.c_int32), C.c_void_p]
    L.gp_set_snapshot_device.restype = C.c_int
    L.gp_set_snapshot_device.argtypes = [C.c_void_p, C.POINTER(gp_nodes), C.c_int32, C.c_int32, C.c_void_p]
    L.gp_pack_batch_device.restype = C.c_int
    L.gp_pack_batch_device.argtypes = [C.c_void_p, C.POINTER(gp_apps), C.c_int, C.c_int, C.POINTER(gp_results), C.c_void_p]
    L.gp_stream.restype = C.c_void_p
    L.gp_stream.argtypes = [C.c_void_p]
    L.gp_synchronize.restype = C.c_int
    L.gp_synchronize.argtypes = [C.c_void_p]
    L.gp_last_stats.restype = C.c_int
    L.gp_last_stats.argtypes = [C.c_void_p, C.POINTER(gp_stats)]
    L.gp_build_availability.restype = C.c_int
    L.gp_build_availability.argtypes = [C.c_void_p, C.POINTER(gp_usage_input)] + [C.c_void_p] * 6
    L.gp_build_reschedule_availability.restype = C.c_int
    L.gp_build_reschedule_availability.argtypes = [C.c_void_p, C.POINTER(gp_usage_input)] + [C.c_void_p] * 3
    L.gp_prepare_cluster.restype = C.c_int
    L.gp_prepare_cluster.argtypes = [C.c_void_p, C.POINTER(gp_usage_input), C.POINTER(gp_sort_input), C.POINTER(C.c_int32),
                                     C.POINTER(C.c_int32)]
    L.gp_prepare_cluster_zones.restype = C.c_int
    L.gp_prepare_cluster_zones.argtypes = [C.c_void_p, C.POINTER(gp_usage_input), C.POINTER(gp_sort_input), C.POINTER(gp_zone_layout)]
    L.gp_prepare_cluster_zones_groups.restype = C.c_int
    L.gp_prepare_cluster_zones_groups.argtypes = [C.c_void_p, C.POINTER(gp_usage_input), C.POINTER(gp_sort_input), C.c_void_p, C.c_int32,
                                                  C.POINTER(gp_instance_group_layout)]
    L.gp_prepare_cluster_groups.restype = C.c_int
    L.gp_prepare_cluster_groups.argtypes = [C.c_void_p, C.POINTER(gp_usage_input), C.POINTER(gp_sort_input), C.c_void_p, C.c_int32,
                                            C.POINTER(gp_instance_group_orders)]
    L.gp_potential_nodes.restype = C.c_int
    L.gp_potential_nodes.argtypes = [C.c_void_p, C.POINTER(gp_sort_input), C.c_void_p, C.POINTER(C.c_int32),
                                     C.c_void_p, C.POINTER(C.c_int32)]
    L.gp_reschedule_executors.restype = C.c_int
    L.gp_reschedule_executors.argtypes = [C.c_void_p, C.POINTER(gp_reschedule), C.c_void_p]
    L.gp_reschedule_from_reservations.restype = C.c_int
    L.gp_reschedule_from_reservations.argtypes = [C.c_void_p, C.POINTER(gp_usage_input), C.POINTER(gp_sort_input),
                                                  C.POINTER(gp_reschedule_scope), C.POINTER(gp_reschedule), C.c_void_p, C.c_void_p]
    L.gp_multi_create.restype = C.c_int
    L.gp_multi_create.argtypes = [C.POINTER(C.c_void_p), C.c_void_p, C.c_int32]
    L.gp_multi_destroy.restype = None
    L.gp_multi_destroy.argtypes = [C.c_void_p]
    L.gp_multi_last_error.restype = C.c_char_p
    L.gp_multi_last_error.argtypes = [C.c_void_p]
    L.gp_multi_size.restype = C.c_int32
    L.gp_multi_size.argtypes = [C.c_void_p]
    L.gp_multi_ctx.restype = C.c_void_p
    L.gp_multi_ctx.argtypes = [C.c_void_p, C.c_int32]
    L.gp_multi_set_snapshot.restype = C.c_int
    L.gp_multi_set_snapshot.argtypes = [C.c_void_p, C.POINTER(gp_nodes)]
    L.gp_multi_pack_batch.restype = C.c_int
    L.gp_multi_pack_batch.argtypes = [C.c_void_p, C.POINTER(gp_apps_wire), C.c_int, C.c_int, C.POINTER(gp_results_wire)]
    L.gp_multi_get_snapshot.restype = C.c_int
    L.gp_multi_get_snapshot.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.gp_multi_group_owner.restype = C.c_int
    L.gp_multi_group_owner.argtypes = [C.c_void_p, C.c_void_p]
    L.gp_driver_table_reset.restype = C.c_int
    L.gp_driver_table_reset.argtypes = [C.c_void_p, C.POINTER(gp_driver_table_size)]
    L.gp_driver_table_update.restype = C.c_int
    L.gp_driver_table_update.argtypes = [C.c_void_p, C.POINTER(gp_driver_delta)]
    L.gp_pack_fifo_driver_table.restype = C.c_int
    L.gp_pack_fifo_driver_table.argtypes = [C.c_void_p, C.POINTER(gp_driver_queue), C.c_int, C.c_int, C.POINTER(gp_results)]
    L.gp_pack_fifo_zones_groups_driver_table.restype = C.c_int
    L.gp_pack_fifo_zones_groups_driver_table.argtypes = [C.c_void_p, C.POINTER(gp_driver_queue), C.c_int, C.c_int, C.c_void_p,
                                                         C.POINTER(gp_zone_results)]
    L.gp_exceeds_cluster_capacity_driver_table.restype = C.c_int
    L.gp_exceeds_cluster_capacity_driver_table.argtypes = [C.c_void_p, C.POINTER(gp_node_table_nodes), C.POINTER(gp_node_affinities),
                                                           C.POINTER(gp_stale_sweep), C.c_int]
    _lib = L
    return L


def _np(a, dtype):
    return None if a is None else np.ascontiguousarray(a, dtype=dtype)


def _p(a):
    return None if a is None else a.ctypes.data


def _triple(t):
    """(cpu, mem[, gpu]) columns, the gpu one absent or None -> three int64 arrays (gpu None when not given)."""
    return [_np(t[i], np.int64) if i < len(t) else None for i in range(3)]


_DT_DELTA_COLS = {"slot": np.int32, "present": np.uint8, "creation": np.int64, "scheduler": np.int32, "group": np.int32,
                  "drv_cpu_milli": np.int64, "drv_mem_bytes": np.int64, "drv_gpu": np.int64, "exe_cpu_milli": np.int64,
                  "exe_mem_bytes": np.int64, "exe_gpu": np.int64, "min_executor_count": np.int32, "exact": np.uint8,
                  "affinity": np.int32}


def _usage_input(alloc, overhead, res_node, res):
    """gp_usage_input over (cpu, mem[, gpu]) triples; overhead may be None.  The struct keeps its arrays alive."""
    al, rs = _triple(alloc), _triple(res)
    ov = _triple(overhead) if overhead is not None else [None] * 3
    rn = _np(res_node, np.int32)
    ui = gp_usage_input(n_nodes=len(al[0]), alloc_cpu_milli=_p(al[0]), alloc_mem_bytes=_p(al[1]), alloc_gpu=_p(al[2]),
                        overhead_cpu_milli=_p(ov[0]), overhead_mem_bytes=_p(ov[1]), overhead_gpu=_p(ov[2]),
                        n_reservations=len(rn), res_node=_p(rn), res_cpu_milli=_p(rs[0]), res_mem_bytes=_p(rs[1]), res_gpu=_p(rs[2]))
    ui._keep = (al, ov, rn, rs)
    return ui


def _resident_usage(node_id, alloc, overhead=None, overhead_node_id=None):
    """gp_resident_usage: node_id[n] reservation-table ids, alloc / overhead (cpu, mem[, gpu]) triples (overhead may be None),
    overhead_node_id[n] overhead-table ids or None (overhead from the host arrays).  The struct keeps its arrays alive."""
    ids, al = _np(node_id, np.int32), _triple(alloc)
    ov = _triple(overhead) if overhead is not None else [None] * 3
    oid = _np(overhead_node_id, np.int32)
    ru = gp_resident_usage(n_nodes=len(ids), node_id=_p(ids), alloc_cpu_milli=_p(al[0]), alloc_mem_bytes=_p(al[1]), alloc_gpu=_p(al[2]),
                           overhead_node_id=_p(oid), overhead_cpu_milli=_p(ov[0]), overhead_mem_bytes=_p(ov[1]), overhead_gpu=_p(ov[2]))
    ru._keep = (ids, al, ov, oid)
    return ru


def _resident_labels(node_id):
    ids = _np(node_id, np.int32)
    rl = gp_resident_labels(n_nodes=len(ids), node_id=_p(ids))
    rl._keep = ids
    return rl


def _node_table_nodes(node_table_id, reservation_id, overhead_node_id, is_driver_candidate=None, zone_key=-1, zone_value=None,
                      n_zones=1, zone_missing=-1, instance_group_key=-1, instance_group_value=None, driver_rank_key=-1,
                      driver_rank_value=None, executor_rank_key=-1, executor_rank_value=None, zone_id_out=None,
                      instance_group_out=None):
    """gp_node_table_nodes (zone_id_out / instance_group_out: int32 arrays the call fills, or None).  The struct keeps its
    arrays alive."""
    tid, rid, oid = _np(node_table_id, np.int32), _np(reservation_id, np.int32), _np(overhead_node_id, np.int32)
    cand = _np(is_driver_candidate, np.uint8)
    zv, igv = _np(zone_value, np.int32), _np(instance_group_value, np.int32)
    drv, exe = _np(driver_rank_value, np.int32), _np(executor_rank_value, np.int32)
    nt = gp_node_table_nodes(n_nodes=len(tid), node_table_id=_p(tid), reservation_id=_p(rid), overhead_node_id=_p(oid),
                             is_driver_candidate=_p(cand), zone_key=int(zone_key), n_zones=int(n_zones), zone_value=_p(zv),
                             zone_missing=int(zone_missing), instance_group_key=int(instance_group_key), instance_group_value=_p(igv),
                             driver_rank_key=int(driver_rank_key), n_driver_rank_values=0 if drv is None else len(drv),
                             driver_rank_value=_p(drv), executor_rank_key=int(executor_rank_key),
                             n_executor_rank_values=0 if exe is None else len(exe), executor_rank_value=_p(exe),
                             zone_id_out=_p(zone_id_out), instance_group_out=_p(instance_group_out))
    nt._keep = (tid, rid, oid, cand, zv, igv, drv, exe, zone_id_out, instance_group_out)
    return nt


def _node_table_entry(entry):
    """The call of a *_node_table entry in the place of its *_resident entry's: the helpers pass (handle, gp_node_table_nodes,
    gp_sort_input, rest...), and the gp_sort_input only lends its undefined_ties."""
    def fn(h, nt_ref, si_ref, *rest):
        nt_ref._obj.undefined_ties = si_ref._obj.undefined_ties
        return entry(h, nt_ref, *rest)
    return fn


def _capacity_nodes(alloc, overhead, zone_id, n_zones, node_group, n_groups):
    """gp_capacity_nodes over (cpu, mem[, gpu]) triples; overhead may be None.  The struct keeps its arrays alive."""
    al = [_np(v, np.int64) for v in alloc]
    ov = [_np(v, np.int64) for v in overhead] if overhead is not None else [None, None, None]
    zid, grp = _np(zone_id, np.int32), _np(node_group, np.int32)
    nd = gp_capacity_nodes(n_nodes=len(al[0]), alloc_cpu_milli=_p(al[0]), alloc_mem_bytes=_p(al[1]),
                           alloc_gpu=_p(al[2] if len(al) > 2 else None), overhead_cpu_milli=_p(ov[0]), overhead_mem_bytes=_p(ov[1]),
                           overhead_gpu=_p(ov[2] if len(ov) > 2 else None), n_zones=int(n_zones), zone_id=_p(zid),
                           n_groups=int(n_groups), node_group=_p(grp))
    nd._keep = (al, ov, zid, grp)
    return nd


def _sort_input(n, n_zones, zone_id=None, name_rank=None, is_driver_candidate=None, unschedulable=None, ready=None,
                driver_label_rank=None, executor_label_rank=None, avail=(None, None, None), ties=None):
    """gp_sort_input over n nodes.  avail: the host (cpu, mem, gpu) availability, None where the availability stage
    supplies it on the device; ties: a c_int32 receiving undefined_ties, or None.  The struct keeps its arrays alive."""
    ids = [_np(zone_id, np.int32), _np(name_rank, np.int32), _np(is_driver_candidate, np.uint8), _np(unschedulable, np.uint8),
           _np(ready, np.uint8), _np(driver_label_rank, np.int32), _np(executor_label_rank, np.int32)]
    av = [_np(x, np.int64) for x in avail]
    si = gp_sort_input(n_nodes=n, avail_cpu_milli=_p(av[0]), avail_mem_bytes=_p(av[1]), n_zones=n_zones, zone_id=_p(ids[0]),
                       name_rank=_p(ids[1]), is_driver_candidate=_p(ids[2]), unschedulable=_p(ids[3]), ready=_p(ids[4]),
                       driver_label_rank=_p(ids[5]), executor_label_rank=_p(ids[6]), avail_gpu=_p(av[2]),
                       undefined_ties=None if ties is None else C.addressof(ties))
    si._keep = (ids, av)
    return si


def _hosting(hosting, q):
    """Per-executor lists of node indices -> the (host_off[q + 1], host_nodes) CSR, or (None, None) without `hosting`."""
    if hosting is None:
        return None, None
    hoff = np.zeros(q + 1, np.int64)
    np.cumsum([len(h) for h in hosting], out=hoff[1:])
    return hoff, np.array([v for h in hosting for v in h] or [0], np.int32)


def _apps(apps, off, group=None, skip=None):
    """gp_apps over the six quantity columns and count of `apps`, with these offsets, group and skip_if_no_fit columns (each
    may be None).  The struct keeps its arrays alive."""
    cols = [_np(apps.get(k), np.int64) for k in ("drv_cpu", "drv_mem", "drv_gpu", "exe_cpu", "exe_mem", "exe_gpu")]
    count, off = _np(apps["count"], np.int32), _np(off, np.int64)
    group, skip = _np(group, np.int32), _np(skip, np.uint8)
    a = gp_apps(n_apps=len(count), drv_cpu_milli=_p(cols[0]), drv_mem_bytes=_p(cols[1]), drv_gpu=_p(cols[2]),
                exe_cpu_milli=_p(cols[3]), exe_mem_bytes=_p(cols[4]), exe_gpu=_p(cols[5]), exe_count=_p(count), group=_p(group),
                skip_if_no_fit=_p(skip), exec_out_off=_p(off))
    a._keep = (cols, count, off, group, skip)
    return a


def _az_orders(exec_order, drv_order, n_zones):
    """-> (pointer argument, kept arrays): a gp_az_orders, or NULL when all three are None (the orders
    prepare_cluster_zones(LAYOUT_AZ_AWARE) left on the device)."""
    if exec_order is None and drv_order is None and n_zones is None:
        return None, None
    eo, do = _np(exec_order, np.int32), _np(drv_order, np.int32)
    o = gp_az_orders(n_zones=int(n_zones), n_exec=len(eo), exec_order=_p(eo), n_drv=len(do), drv_order=_p(do))
    return C.byref(o), (o, eo, do)


def _instance_groups(group_off, n_zones=None, exec_off=None, exec_order=None, drv_off=None, drv_order=None):
    """-> (gp_instance_groups, kept arrays) over int32 copies of the given columns (None stays NULL)."""
    cols = [_np(x, np.int32) for x in (group_off, n_zones, exec_off, exec_order, drv_off, drv_order)]
    ig = gp_instance_groups(len(cols[0]) - 1, *[_p(x) for x in cols])
    return ig, cols


_LABEL_COLS = {"label_off": np.int64, "label_key": np.int32, "label_val": np.int32, "label_int_ok": np.uint8, "label_int": np.int64}
_AFF_COLS = {"sel_off": np.int64, "sel_key": np.int32, "sel_val": np.int32, "has_required": np.uint8, "term_off": np.int64,
             "term_req_off": np.int64, "term_parse_error": np.uint8, "req_op": np.int32, "req_key": np.int32, "req_int": np.int64,
             "req_val_off": np.int64, "req_val": np.int32}


# gp_overhead_delta's columns (overhead.OverheadTable.delta() keys)
_DELTA_COLS = {"slot": np.int32, "node_id": np.int32, "req_cpu_milli": np.int64, "req_mem_bytes": np.int64, "req_gpu": np.int64,
               "listed": np.uint8, "app_key": np.int32, "app_id": np.int32, "name_id": np.int32, "is_executor": np.uint8,
               "spark_scheduler": np.uint8, "rr_app_key": np.int32, "rr_exists": np.uint8, "member_kind": np.uint8,
               "member_app": np.int32, "member_name": np.int32, "member_present": np.uint8}

# gp_label_delta's columns (affinity.LabelTable.delta() keys)
_LT_DELTA_COLS = {"row_node": np.int32, "row_off": np.int64, "label_key": np.int32, "label_val": np.int32, "value_id": np.int32,
                  "value_int_ok": np.uint8, "value_int": np.int64}

# gp_node_delta's columns (nodes.NodeTable.delta() keys)
_NT_DELTA_COLS = {"node_id": np.int32, "present": np.uint8, "alloc_cpu_milli": np.int64, "alloc_mem_bytes": np.int64,
                  "alloc_gpu": np.int64, "unschedulable": np.uint8, "ready": np.uint8, "name_key": np.int64, "creation": np.int64}

# gp_reservation_delta's columns (reservations.ReservationTable.delta() keys)
_RT_DELTA_COLS = {"slot": np.int32, "node_id": np.int32, "cpu_milli": np.int64, "mem_bytes": np.int64, "gpu": np.int64}

_OVERHEAD_COLS = {"node_id": np.int32, "req_cpu_milli": np.int64, "req_mem_bytes": np.int64, "req_gpu": np.int64, "listed": np.uint8,
                  "app_key": np.int32, "app_id": np.int32, "name_id": np.int32, "is_executor": np.uint8, "spark_scheduler": np.uint8,
                  "rr_app_key": np.int32, "rr_pod_off": np.int64, "rr_pod_name": np.int32, "soft_app_id": np.int32,
                  "soft_pod_off": np.int64, "soft_pod_name": np.int32, "node_ids": np.int32}


def _affinity_input(enc: dict):
    """(gp_node_labels, gp_node_affinities) over the arrays of affinity.encode() (or the same keys given by hand; a missing
    optional column is NULL).  The structs keep their arrays alive."""
    lc = {k: _np(enc.get(k), t) for k, t in _LABEL_COLS.items()}
    n = int(enc["n_nodes"]) if "n_nodes" in enc else len(lc["label_off"]) - 1
    lab = gp_node_labels(n_nodes=n, n_keys=int(enc["n_keys"]), n_values=int(enc["n_values"]), **{k: _p(v) for k, v in lc.items()})
    lab._keep = lc
    return lab, _programs(enc)


def _programs(enc: dict):
    """gp_node_affinities over the program arrays of enc; the struct keeps its arrays alive."""
    ac = {k: _np(enc.get(k), t) for k, t in _AFF_COLS.items()}
    n_aff = int(enc["n_aff"]) if "n_aff" in enc else len(ac["sel_off"]) - 1
    aff = gp_node_affinities(n_aff=n_aff, **{k: _p(v) for k, v in ac.items()})
    aff._keep = ac
    return aff


def compact_apps(apps: dict, mem_shift: int = 20):
    """What the shim does while marshalling: the 32-bit wire layout when every quantity is exactly representable
    (memory a whole multiple of 2^mem_shift bytes, everything < 2^31), else None (use the int64 layout)."""
    out = dict(apps)
    for k in ("drv_cpu", "drv_gpu", "exe_cpu", "exe_gpu", "drv_mem", "exe_mem"):
        v = apps.get(k)
        if v is None:
            continue
        v = np.asarray(v, np.int64)
        if k.endswith("mem"):
            if (v & ((1 << mem_shift) - 1)).any():
                return None
            v = v >> mem_shift
        if (v < 0).any() or (v >= (1 << 31)).any():
            return None
        out[k] = v.astype(np.int32)
    return out


class PinnedArray:
    """numpy view over gp_alloc_pinned memory."""

    def __init__(self, packer: "GangPacker", shape, dtype):
        self._packer = packer
        self.dtype = np.dtype(dtype)
        n = int(np.prod(shape)) if np.ndim(shape) else int(shape)
        self.nbytes = max(n * self.dtype.itemsize, 1)
        ptr = C.c_void_p()
        packer._check(load().gp_alloc_pinned(packer._h, self.nbytes, C.byref(ptr)))
        self._ptr = ptr
        buf = (C.c_char * self.nbytes).from_address(ptr.value)
        self.array = np.frombuffer(buf, dtype=self.dtype, count=n).reshape(shape)

    def free(self):
        if self._ptr is not None and self._packer._h:
            self.array = None
            load().gp_free_pinned(self._packer._h, self._ptr)
            self._ptr = None


class GangPacker:
    """One gp_ctx.  Not thread-safe (like the C ABI)."""

    def __init__(self, device: int = -1, async_snapshot: bool = False):
        L = load()
        self._h = C.c_void_p()
        cfg = gp_config(device=device, flags=CFG_ASYNC_SNAPSHOT if async_snapshot else 0)
        st = L.gp_create(C.byref(self._h), C.byref(cfg))
        if st != 0:
            raise GangpackError(st, (L.gp_last_error(None) or b"").decode())
        self._keep = None
        self._pinned = []
        self._registered = []

    def close(self):
        if getattr(self, "_h", None):
            for p in self._pinned:
                p.free()
            self._pinned = []
            for addr in self._registered:
                load().gp_unregister_host(self._h, addr)
            self._registered = []
            load().gp_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, st: int):
        if st != 0:
            raise GangpackError(st, (load().gp_last_error(self._h) or b"").decode())

    def pinned(self, shape, dtype) -> np.ndarray:
        p = PinnedArray(self, shape, dtype)
        self._pinned.append(p)
        return p.array

    def register_host(self, array: np.ndarray):
        """Page-lock caller-owned memory (e.g. a shared-memory segment) so results can be DMA'd straight into it."""
        self._check(load().gp_register_host(self._h, array.ctypes.data, array.nbytes))
        self._registered.append(array.ctypes.data)

    def unregister_host(self, array: np.ndarray):
        self._check(load().gp_unregister_host(self._h, array.ctypes.data))
        self._registered.remove(array.ctypes.data)

    def pinned_columns(self, n: int, names, dtype=np.int64) -> dict:
        """`names` equally spaced columns of n elements inside ONE pinned block (column after column): the layout
        that lets gp_pack_batch move all int64 columns of a chunk with a single 2-D DMA."""
        block = self.pinned((len(names), n), dtype)
        return {name: block[i] for i, name in enumerate(names)}

    # ---- snapshot ----------------------------------------------------------------------------
    def set_snapshot(self, avail_cpu, avail_mem, avail_gpu, exec_order, drv_order, exec_off=None, drv_off=None):
        cpu, mem = _np(avail_cpu, np.int64), _np(avail_mem, np.int64)
        gpu = _np(avail_gpu, np.int64)
        eo, do = _np(exec_order, np.int32), _np(drv_order, np.int32)
        eoff = _np(exec_off if exec_off is not None else [0, len(eo)], np.int32)
        doff = _np(drv_off if drv_off is not None else [0, len(do)], np.int32)
        n = gp_nodes(n_nodes=len(cpu), avail_cpu_milli=_p(cpu), avail_mem_bytes=_p(mem), avail_gpu=_p(gpu),
                     n_groups=len(eoff) - 1, exec_off=_p(eoff), exec_order=_p(eo), drv_off=_p(doff), drv_order=_p(do))
        self._check(load().gp_set_snapshot(self._h, C.byref(n)))
        self.n_nodes = len(cpu)

    def get_snapshot(self):
        cpu = np.empty(self.n_nodes, np.int64); mem = np.empty(self.n_nodes, np.int64); gpu = np.empty(self.n_nodes, np.int64)
        self._check(load().gp_get_snapshot(self._h, _p(cpu), _p(mem), _p(gpu)))
        return cpu, mem, gpu

    # ---- executors without a usable reservation (rescheduleExecutor's node choice) -----------------
    def reschedule_executors(self, exe, min_frag=False, group=None, reserved=None, hosting=None):
        """exe: (cpu[q], mem[q], gpu[q]|None); reserved: (cpu[n], mem[n], gpu[n]|None) or None; hosting: list of
        per-executor node-index lists (nodes already hosting executors of the same application) or None.
        -> node index per executor (-1: no capacity)."""
        ec, em = _np(exe[0], np.int64), _np(exe[1], np.int64)
        eg = _np(exe[2], np.int64) if len(exe) > 2 else None
        q = len(ec)
        grp = _np(group, np.int32)
        rs = [_np(x, np.int64) for x in reserved] if reserved is not None else [None] * 3
        hoff, hn = _hosting(hosting, q)
        out = np.full(max(q, 1), -9, np.int32)
        r = gp_reschedule(n_execs=q, exe_cpu_milli=_p(ec), exe_mem_bytes=_p(em), exe_gpu=_p(eg), group=_p(grp),
                          min_frag=1 if min_frag else 0, reserved_cpu_milli=_p(rs[0]), reserved_mem_bytes=_p(rs[1]),
                          reserved_gpu=_p(rs[2] if len(rs) > 2 else None), host_off=_p(hoff), host_nodes=_p(hn))
        self._check(load().gp_reschedule_executors(self._h, C.byref(r), _p(out)))
        return out[:q]

    # ---- availability snapshot from reservations (NodeSchedulingMetadataForNodes) ----------------
    def build_availability(self, alloc, overhead, res_node, res):
        """alloc / overhead / res: (cpu, mem, gpu) triples (overhead may be None) -> (avail triple, sched triple).
        Exact or refused: |allocatable|, |overhead|, a counted |reservation|, a node's exact reservation sum or a result
        >= 2^61 raises GangpackError with GP_ERR_UNREPRESENTABLE; nothing is computed modulo 2^64."""
        ui = _usage_input(alloc, overhead, res_node, res)
        n = ui.n_nodes
        outs = [np.empty(max(n, 1), np.int64) for _ in range(6)]
        self._check(load().gp_build_availability(self._h, C.byref(ui), *[_p(o) for o in outs]))
        return [o[:n] for o in outs[:3]], [o[:n] for o in outs[3:]]

    def build_reschedule_availability(self, alloc, overhead, res_node, res):
        """availableResources of rescheduleExecutor's first-fit branch (overhead counted twice on nodes with a reservation row,
        whatever its resources).  The domain and its refusal as in build_availability."""
        ui = _usage_input(alloc, overhead, res_node, res)
        n = ui.n_nodes
        outs = [np.empty(max(n, 1), np.int64) for _ in range(3)]
        self._check(load().gp_build_reschedule_availability(self._h, C.byref(ui), *[_p(o) for o in outs]))
        return [o[:n] for o in outs]

    def reschedule_from_reservations(self, alloc, overhead, res_node, res, exe, min_frag=False, hosting=None, zone_id=None,
                                     n_zones=1, name_rank=None, unschedulable=None, ready=None, executor_label_rank=None,
                                     keep_topology_zone=None, topology_zone=None):
        """rescheduleExecutor from the reservations to the node choice in one device call, for a batch of executors.
        alloc / overhead / res / exe: (cpu, mem, gpu) triples (overhead and the gpu entries may be None); hosting: per-executor
        lists of node indices already hosting executors of the same application, or None; keep_topology_zone: None (every
        node) or the zone id filterNodesToZone keeps, with topology_zone[n] the node's zone id (-1 = label missing).
        The context's snapshot is not touched.  The domain and its refusal as in build_availability; name_rank must be a
        permutation (GP_ERR_INVALID).  -> (node index per executor or -1, ambiguous flag per executor)."""
        return self._reschedule(load().gp_reschedule_from_reservations, _usage_input(alloc, overhead, res_node, res), exe, min_frag,
                                hosting, zone_id, n_zones, name_rank, unschedulable, ready, executor_label_rank, keep_topology_zone,
                                topology_zone)

    def reschedule_from_reservations_resident(self, node_id, alloc, overhead, exe, min_frag=False, hosting=None, zone_id=None,
                                              n_zones=1, name_rank=None, unschedulable=None, ready=None, executor_label_rank=None,
                                              keep_topology_zone=None, topology_zone=None, overhead_node_id=None):
        """reschedule_from_reservations with the reservations from the resident reservation table: node_id[n] = each node's
        reservation-table id (-1 = none); overhead from the host triple (or None), or with overhead_node_id[n] from the
        resident overhead table.  Returns what reschedule_from_reservations returns on the equivalent rows."""
        return self._reschedule(load().gp_reschedule_from_reservations_resident, _resident_usage(node_id, alloc, overhead, overhead_node_id),
                                exe, min_frag, hosting, zone_id, n_zones, name_rank, unschedulable, ready, executor_label_rank,
                                keep_topology_zone, topology_zone)

    def _reschedule(self, fn, ui, exe, min_frag, hosting, zone_id, n_zones, name_rank, unschedulable, ready, executor_label_rank,
                    keep_topology_zone, topology_zone):
        n = ui.n_nodes
        si = _sort_input(n, n_zones, zone_id=zone_id, name_rank=name_rank, unschedulable=unschedulable, ready=ready,
                         executor_label_rank=executor_label_rank)
        tz = _np(topology_zone, np.int32)
        scope = None
        if keep_topology_zone is not None:
            scope = gp_reschedule_scope(keep_topology_zone=int(keep_topology_zone), topology_zone=_p(tz))
        ec, em = _np(exe[0], np.int64), _np(exe[1], np.int64)
        eg = _np(exe[2], np.int64) if len(exe) > 2 else None
        q = len(ec)
        hoff, hn = _hosting(hosting, q)
        r = gp_reschedule(n_execs=q, exe_cpu_milli=_p(ec), exe_mem_bytes=_p(em), exe_gpu=_p(eg), min_frag=1 if min_frag else 0,
                          host_off=_p(hoff), host_nodes=_p(hn))
        out = np.full(max(q, 1), -9, np.int32)
        amb = np.full(max(q, 1), 9, np.uint8)
        self._check(fn(self._h, C.byref(ui), C.byref(si), C.byref(scope) if scope is not None else None, C.byref(r), _p(out), _p(amb)))
        return out[:q], amb[:q]

    def prepare_cluster(self, alloc, overhead, res_node, res, zone_id=None, n_zones=1, name_rank=None, is_driver_candidate=None,
                        unschedulable=None, ready=None, driver_label_rank=None, executor_label_rank=None):
        """reservations -> availability -> priority orders -> snapshot, chained on the device.  -> (n_driver, n_executor).
        A quantity, reservation sum or availability outside the exact-int64 domain (|v| >= 2^61) raises GangpackError
        (GP_ERR_UNREPRESENTABLE) and the snapshot the context held stays in place."""
        ui = _usage_input(alloc, overhead, res_node, res)
        n = ui.n_nodes
        si = _sort_input(n, n_zones, zone_id, name_rank, is_driver_candidate, unschedulable, ready, driver_label_rank,
                         executor_label_rank)
        nd, ne = C.c_int32(0), C.c_int32(0)
        self._check(load().gp_prepare_cluster(self._h, C.byref(ui), C.byref(si), C.byref(nd), C.byref(ne)))
        self.n_nodes = n
        return nd.value, ne.value

    def prepare_cluster_zones(self, alloc, overhead, res_node, res, zone_id=None, n_zones=1, name_rank=None, is_driver_candidate=None,
                              unschedulable=None, ready=None, driver_label_rank=None, executor_label_rank=None, kind=LAYOUT_AZ_AWARE,
                              layout=True):
        """reservations -> availability -> priority orders -> zone-grouped snapshot (kind LAYOUT_SINGLE_AZ or LAYOUT_AZ_AWARE),
        chained on the device, SchedulableResources included.  -> dict with n_zones, n_groups, n_driver, n_executor,
        zone_of_group, undefined_ties and, with `layout`, the grouped exec_off / exec_order / drv_off / drv_order.
        The domain and its refusal as in prepare_cluster: a refused call leaves the context as it was."""
        ui = _usage_input(alloc, overhead, res_node, res)
        n = ui.n_nodes
        ties = C.c_int32(0)
        si = _sort_input(n, n_zones, zone_id, name_rank, is_driver_candidate, unschedulable, ready, driver_label_rank,
                         executor_label_rank, ties=ties)
        zog = np.full(n_zones + 1, -9, np.int32)
        bufs = {k: np.full(max(n, 1) if k.endswith("order") else n_zones + 2, -9, np.int32)
                for k in ("exec_off", "exec_order", "drv_off", "drv_order")} if layout else {}
        lo = gp_zone_layout(kind=int(kind), zone_of_group=_p(zog), **{k: _p(v) for k, v in bufs.items()})
        self._check(load().gp_prepare_cluster_zones(self._h, C.byref(ui), C.byref(si), C.byref(lo)))
        self.n_nodes = n
        out = dict(n_zones=lo.n_zones, n_groups=lo.n_groups, n_driver=lo.n_driver, n_executor=lo.n_executor, zone_of_group=zog,
                   undefined_ties=ties.value)
        if layout:
            G = lo.n_groups
            out.update(exec_off=bufs["exec_off"][:G + 1].copy(), drv_off=bufs["drv_off"][:G + 1].copy())
            out.update(exec_order=bufs["exec_order"][:out["exec_off"][G]].copy(), drv_order=bufs["drv_order"][:out["drv_off"][G]].copy())
        return out

    def prepare_cluster_zones_groups(self, alloc, overhead, res_node, res, instance_group, n_instance_groups, zone_id=None, n_zones=1,
                                     name_rank=None, is_driver_candidate=None, unschedulable=None, ready=None, driver_label_rank=None,
                                     executor_label_rank=None, kind=LAYOUT_AZ_AWARE, layout=True):
        """prepare_cluster_zones for every instance group at once: instance_group[v] = node v's instance group (0 ..
        n_instance_groups-1, -1 = none; None = every node in 0).  Each instance group's orders are PotentialNodes over its own
        nodes, grouped by zone; its groups follow those of the instance groups before it.  -> dict with n_groups, n_driver,
        n_executor, undefined_ties (the total), group_off, n_zones, exec_off, drv_off, ig_undefined_ties (per instance group)
        and, with `layout`, the undivided exec_order / drv_order, the grouped group_exec_off / group_exec_order /
        group_drv_off / group_drv_order and zone_of_group.  The context then holds the layout pack_fifo_zones_groups drains
        when its layout arguments are all None.  A refused call leaves the context as it was."""
        return self._prepare_zones_groups(load().gp_prepare_cluster_zones_groups, _usage_input(alloc, overhead, res_node, res),
                                          instance_group, n_instance_groups, zone_id, n_zones, name_rank, is_driver_candidate,
                                          unschedulable, ready, driver_label_rank, executor_label_rank, kind, layout)

    def prepare_cluster_zones_groups_resident(self, node_id, alloc, overhead, instance_group, n_instance_groups, zone_id=None, n_zones=1,
                                              name_rank=None, is_driver_candidate=None, unschedulable=None, ready=None,
                                              driver_label_rank=None, executor_label_rank=None, kind=LAYOUT_AZ_AWARE, layout=True,
                                              overhead_node_id=None):
        """prepare_cluster_zones_groups with the reservations from the resident reservation table (node_id, overhead and
        overhead_node_id as in reschedule_from_reservations_resident).  Returns what prepare_cluster_zones_groups returns on
        the equivalent rows, and leaves the context as it would."""
        return self._prepare_zones_groups(load().gp_prepare_cluster_zones_groups_resident,
                                          _resident_usage(node_id, alloc, overhead, overhead_node_id), instance_group, n_instance_groups,
                                          zone_id, n_zones, name_rank, is_driver_candidate, unschedulable, ready, driver_label_rank,
                                          executor_label_rank, kind, layout)

    def _prepare_zones_groups(self, fn, ui, instance_group, n_instance_groups, zone_id, n_zones, name_rank, is_driver_candidate,
                              unschedulable, ready, driver_label_rank, executor_label_rank, kind, layout):
        n = ui.n_nodes
        G = int(n_instance_groups)
        ig = _np(instance_group, np.int32)
        ties = C.c_int32(0)
        si = _sort_input(n, n_zones, zone_id, name_rank, is_driver_candidate, unschedulable, ready, driver_label_rank,
                         executor_label_rank, ties=ties)
        g1 = max(G, 0) + 1
        bufs = {k: np.full(g1, -9, np.int32) for k in ("group_off", "n_zones", "exec_off", "drv_off", "undefined_ties")}
        if layout:
            n_groups_max = g1 + min(n, max(G, 0) * n_zones)
            bufs.update({k: np.full(max(n, 1), -9, np.int32) for k in ("exec_order", "drv_order", "group_exec_order", "group_drv_order")})
            bufs.update({k: np.full(n_groups_max + 1, -9, np.int32) for k in ("group_exec_off", "group_drv_off", "zone_of_group")})
        lo = gp_instance_group_layout(kind=int(kind), **{k: _p(v) for k, v in bufs.items()})
        self._check(fn(self._h, C.byref(ui), C.byref(si), _p(ig), G, C.byref(lo)))
        self.n_nodes = n
        out = dict(n_groups=lo.n_groups, n_driver=lo.n_driver, n_executor=lo.n_executor, undefined_ties=ties.value,
                   group_off=bufs["group_off"].copy(), n_zones=bufs["n_zones"][:G].copy(), exec_off=bufs["exec_off"].copy(),
                   drv_off=bufs["drv_off"].copy(), ig_undefined_ties=bufs["undefined_ties"][:G].copy())
        if layout:
            ng = lo.n_groups
            out.update(exec_order=bufs["exec_order"][:lo.n_executor].copy(), drv_order=bufs["drv_order"][:lo.n_driver].copy(),
                       group_exec_off=bufs["group_exec_off"][:ng + 1].copy(), group_drv_off=bufs["group_drv_off"][:ng + 1].copy(),
                       zone_of_group=bufs["zone_of_group"][:ng].copy())
            out.update(group_exec_order=bufs["group_exec_order"][:out["group_exec_off"][ng]].copy(),
                       group_drv_order=bufs["group_drv_order"][:out["group_drv_off"][ng]].copy())
        return out

    def prepare_cluster_groups(self, alloc, overhead, res_node, res, instance_group, n_instance_groups, zone_id=None, n_zones=1,
                               name_rank=None, is_driver_candidate=None, unschedulable=None, ready=None, driver_label_rank=None,
                               executor_label_rank=None, orders=True):
        """prepare_cluster for every instance group at once: instance_group[v] = node v's instance group (0 ..
        n_instance_groups-1, -1 = none; None = every node in 0).  Snapshot group i holds instance group i's PotentialNodes
        orders over its own nodes, ready for pack_batch with apps["group"] = the instance group.  -> dict with n_driver,
        n_executor, undefined_ties (the total), ig_undefined_ties (per instance group) and, with `orders`, exec_off / drv_off
        ([n_instance_groups + 1]) and the instance-group-major exec_order / drv_order.  A refused call leaves the context as
        it was."""
        return self._prepare_groups(load().gp_prepare_cluster_groups, _usage_input(alloc, overhead, res_node, res), instance_group,
                                    n_instance_groups, zone_id, n_zones, name_rank, is_driver_candidate, unschedulable, ready,
                                    driver_label_rank, executor_label_rank, orders)

    def prepare_cluster_groups_resident(self, node_id, alloc, overhead, instance_group, n_instance_groups, zone_id=None, n_zones=1,
                                        name_rank=None, is_driver_candidate=None, unschedulable=None, ready=None, driver_label_rank=None,
                                        executor_label_rank=None, orders=True, overhead_node_id=None):
        """prepare_cluster_groups with the reservations from the resident reservation table (node_id, overhead and
        overhead_node_id as in reschedule_from_reservations_resident).  Returns what prepare_cluster_groups returns on the
        equivalent rows, and leaves the context as it would."""
        return self._prepare_groups(load().gp_prepare_cluster_groups_resident, _resident_usage(node_id, alloc, overhead, overhead_node_id),
                                    instance_group, n_instance_groups, zone_id, n_zones, name_rank, is_driver_candidate, unschedulable,
                                    ready, driver_label_rank, executor_label_rank, orders)

    def _prepare_groups(self, fn, ui, instance_group, n_instance_groups, zone_id, n_zones, name_rank, is_driver_candidate, unschedulable,
                        ready, driver_label_rank, executor_label_rank, orders):
        n = ui.n_nodes
        G = int(n_instance_groups)
        ig = _np(instance_group, np.int32)
        ties = C.c_int32(0)
        si = _sort_input(n, n_zones, zone_id, name_rank, is_driver_candidate, unschedulable, ready, driver_label_rank,
                         executor_label_rank, ties=ties)
        bufs = {"undefined_ties": np.full(max(G, 0) + 1, -9, np.int32)}
        if orders:
            bufs.update({k: np.full(max(G, 0) + 1, -9, np.int32) for k in ("exec_off", "drv_off")})
            bufs.update({k: np.full(max(n, 1), -9, np.int32) for k in ("exec_order", "drv_order")})
        o = gp_instance_group_orders(**{k: _p(v) for k, v in bufs.items()})
        self._check(fn(self._h, C.byref(ui), C.byref(si), _p(ig), G, C.byref(o)))
        self.n_nodes = n
        out = dict(n_driver=o.n_driver, n_executor=o.n_executor, undefined_ties=ties.value,
                   ig_undefined_ties=bufs["undefined_ties"][:G].copy())
        if orders:
            out.update(exec_off=bufs["exec_off"].copy(), drv_off=bufs["drv_off"].copy(),
                       exec_order=bufs["exec_order"][:o.n_executor].copy(), drv_order=bufs["drv_order"][:o.n_driver].copy())
        return out

    # ---- node priority order (NodeSorter.PotentialNodes) ---------------------------------------
    def potential_nodes(self, avail_cpu, avail_mem, zone_id=None, n_zones=1, name_rank=None, is_driver_candidate=None,
                        unschedulable=None, ready=None, driver_label_rank=None, executor_label_rank=None, avail_gpu=None):
        """-> (driver_order, executor_order) as int32 node-index arrays.  With avail_gpu given, self.undefined_ties is the
        number of adjacent pairs the reference's comparator leaves undefined (SURVEY App. B6).  Any int64 availability is
        ordered exactly (zone totals included); name_rank must be a permutation of 0..n-1 (GP_ERR_INVALID)."""
        n = len(avail_cpu)
        ties = C.c_int32(0)
        si = _sort_input(n, n_zones, zone_id, name_rank, is_driver_candidate, unschedulable, ready, driver_label_rank,
                         executor_label_rank, avail=(avail_cpu, avail_mem, avail_gpu), ties=ties)
        d = np.empty(max(n, 1), np.int32); e = np.empty(max(n, 1), np.int32)
        nd, ne = C.c_int32(0), C.c_int32(0)
        self._check(load().gp_potential_nodes(self._h, C.byref(si), _p(d), C.byref(nd), _p(e), C.byref(ne)))
        self.undefined_ties = ties.value
        return d[:nd.value].copy(), e[:ne.value].copy()

    # ---- packing -----------------------------------------------------------------------------
    def pack_batch(self, apps: dict, algo: int, mode: int = MODE_INDEPENDENT, out=None, wire=None):
        """apps: dict with drv_cpu, drv_mem, [drv_gpu], exe_cpu, exe_mem, [exe_gpu], count, [group], [young],
        [off].  Returns (driver_node[q], executor_nodes[sum count], off[q+1]).

        wire=None: the int64 layout through gp_pack_batch.  wire=dict(quantity_bits=32|64, mem_shift=.., node_bits=16|32,
        offsets=True|False) goes through gp_pack_batch_wire: with quantity_bits 32 the six quantity arrays of `apps` must
        ALREADY be int32 in wire units (millicores, bytes >> mem_shift, gpu units -- see compact_apps()); offsets=False
        passes exec_out_off = NULL (derived on the device)."""
        q = len(apps["count"])
        count = _np(apps["count"], np.int32)
        off = _np(apps.get("off"), np.int64)
        derive = wire is not None and not wire.get("offsets", True)
        if off is None and not (derive and out is not None):      # hot path (caller's buffers, device-derived offsets): no host cumsum
            off = np.zeros(q + 1, np.int64)
            np.cumsum(np.maximum(count, 0), out=off[1:])
        bits = 64 if wire is None else int(wire.get("quantity_bits", 64))
        qdt = np.int64 if bits == 64 else np.int32
        arrs = dict(
            drv_cpu=_np(apps["drv_cpu"], qdt), drv_mem=_np(apps["drv_mem"], qdt),
            drv_gpu=_np(apps.get("drv_gpu"), qdt),
            exe_cpu=_np(apps["exe_cpu"], qdt), exe_mem=_np(apps["exe_mem"], qdt),
            exe_gpu=_np(apps.get("exe_gpu"), qdt),
            group=_np(apps.get("group"), np.int32), young=_np(apps.get("young"), np.uint8))
        total = (int(off[-1]) if q else 0) if off is not None else len(out[1])
        node_bits = 32 if wire is None else int(wire.get("node_bits", 32))
        if out is None:
            driver_node = np.full(q, -9, np.int32)
            executor_nodes = np.full(max(total, 1), -9 if node_bits == 32 else 65535, np.int32 if node_bits == 32 else np.uint16)
        else:
            driver_node, executor_nodes = out
        if wire is None:
            a = gp_apps(n_apps=q, drv_cpu_milli=_p(arrs["drv_cpu"]), drv_mem_bytes=_p(arrs["drv_mem"]),
                        drv_gpu=_p(arrs["drv_gpu"]), exe_cpu_milli=_p(arrs["exe_cpu"]), exe_mem_bytes=_p(arrs["exe_mem"]),
                        exe_gpu=_p(arrs["exe_gpu"]), exe_count=_p(count), group=_p(arrs["group"]),
                        skip_if_no_fit=_p(arrs["young"]), exec_out_off=_p(off))
            r = gp_results(driver_node=_p(driver_node), executor_nodes=_p(executor_nodes),
                           executor_nodes_cap=len(executor_nodes))
            self._check(load().gp_pack_batch(self._h, C.byref(a), algo, mode, C.byref(r)))
        else:
            a = gp_apps_wire(n_apps=q, quantity_bits=bits, mem_shift=int(wire.get("mem_shift", 0)),
                             drv_cpu=_p(arrs["drv_cpu"]), drv_mem=_p(arrs["drv_mem"]), drv_gpu=_p(arrs["drv_gpu"]),
                             exe_cpu=_p(arrs["exe_cpu"]), exe_mem=_p(arrs["exe_mem"]), exe_gpu=_p(arrs["exe_gpu"]),
                             exe_count=_p(count), group=_p(arrs["group"]), skip_if_no_fit=_p(arrs["young"]),
                             exec_out_off=None if derive else _p(off))
            r = gp_results_wire(driver_node=_p(driver_node), executor_nodes=_p(executor_nodes),
                                executor_nodes_cap=len(executor_nodes), node_bits=node_bits)
            self._check(load().gp_pack_batch_wire(self._h, C.byref(a), algo, mode, C.byref(r)))
        return driver_node, executor_nodes[:total], off

    def set_schedulable(self, sched_cpu, sched_mem, sched_gpu=None):
        """NodeSchedulingMetadata.SchedulableResources of the current snapshot's nodes (needed by pack_batch_zones)."""
        c, m, g = _np(sched_cpu, np.int64), _np(sched_mem, np.int64), _np(sched_gpu, np.int64)
        self._check(load().gp_set_schedulable(self._h, _p(c), _p(m), _p(g)))

    def _pack_zones(self, apps: dict, skip, fn, *args, group=None):
        """The zone packs' shared body: fn(ctx, apps, *args, results) -> (zone, driver_node, executor_nodes, off, avg_efficiency)."""
        q = len(apps["count"])
        off = np.zeros(q + 1, np.int64)
        np.cumsum(np.maximum(_np(apps["count"], np.int32), 0), out=off[1:])
        total = int(off[-1]) if q else 0
        zone = np.full(q, -9, np.int32); drv = np.full(q, -9, np.int32)
        exe = np.full(max(total, 1), -9, np.int32); avg = np.zeros((max(q, 1), 4), np.float64)
        a = _apps(apps, off, group=group, skip=skip)
        r = gp_zone_results(zone=_p(zone), driver_node=_p(drv), executor_nodes=_p(exe), executor_nodes_cap=len(exe), avg_efficiency=_p(avg))
        self._check(fn(self._h, C.byref(a), *args, C.byref(r)))
        return zone, drv, exe[:total], off, avg[:q]

    def pack_batch_zones(self, apps: dict, algo: int):
        """single-az-tightly-pack / single-az-minimal-fragmentation for a batch: the snapshot's instance groups are the
        candidate zones.  -> (zone[q], driver_node[q], executor_nodes, off[q+1], avg_efficiency[q,4])."""
        return self._pack_zones(apps, None, load().gp_pack_batch_zones, algo)

    def pack_fifo_zones(self, apps: dict, algo: int, mode: int = 1):
        """fitEarlierDrivers with a single-AZ packer in one launch: `apps` is the queue in order (optional "young" = skip the
        driver instead of blocking the queue when it fits nowhere).  -> like pack_batch_zones; driver_node -2 = never evaluated."""
        return self._pack_zones(apps, apps.get("young"), load().gp_pack_fifo_zones, algo, mode)

    def pack_fifo_az_aware(self, apps: dict, mode: int, exec_order=None, drv_order=None, n_zones=None):
        """fitEarlierDrivers with az-aware-tightly-pack in one launch.  The snapshot's groups 0..n_zones-1 are the candidate
        zones, the groups after them the remaining nodes; exec_order / drv_order are the undivided priority orders (node
        indices) of the fallback -- all three None (orders == NULL): the ones prepare_cluster_zones(LAYOUT_AZ_AWARE) left on
        the device.  -> like pack_fifo_zones; zone -1 with driver_node >= 0 = placed by the fallback."""
        o, _keep = _az_orders(exec_order, drv_order, n_zones)
        return self._pack_zones(apps, apps.get("young"), load().gp_pack_fifo_az_aware, mode, o)

    def pack_batch_az_aware(self, apps: dict, exec_order=None, drv_order=None, n_zones=None):
        """az-aware-tightly-pack for a batch of independent decisions against the unmodified snapshot, in one call.  The
        snapshot layout is that of pack_fifo_az_aware (any n_zones up to the number of groups); exec_order / drv_order are
        the undivided priority orders (node indices) of the fallback, or all three None as in pack_fifo_az_aware.
        -> like pack_batch_zones; zone -1 with driver_node >= 0 = placed by the fallback (zero averages)."""
        o, _keep = _az_orders(exec_order, drv_order, n_zones)
        return self._pack_zones(apps, None, load().gp_pack_batch_az_aware, o)

    def pack_fifo_zones_groups(self, apps: dict, packer: int, mode: int, group_off=None, n_zones=None, exec_off=None, exec_order=None,
                               drv_off=None, drv_order=None):
        """fitEarlierDrivers of every instance group in one launch, one CTA per instance group, with packer
        BP_SINGLE_AZ_TIGHTLY_PACK / BP_SINGLE_AZ_MINIMAL_FRAGMENTATION (instance group i's snapshot groups group_off[i] ..
        group_off[i+1]-1 are its zones) or BP_AZ_AWARE_TIGHTLY_PACK (the first n_zones[i] of them its zones, the rest its
        trailing group; exec_order / drv_order its undivided orders in CSR by exec_off / drv_off).  apps["group"] is each
        application's instance group (absent: 0), "young" as in pack_fifo_zones.  -> like pack_fifo_zones, with zone local to
        the application's instance group.  All six layout arguments None (groups == NULL): the layout
        prepare_cluster_zones_groups left on the device."""
        cols = (group_off, n_zones, exec_off, exec_order, drv_off, drv_order)
        ig, _keep = _instance_groups(*cols) if any(x is not None for x in cols) else (None, None)
        return self._pack_zones(apps, apps.get("young"), load().gp_pack_fifo_zones_groups, packer, mode,
                                C.byref(ig) if ig is not None else None, group=apps.get("group"))

    def reserve_placements(self, apps: dict, placed, subtract=True):
        """newResourceReservation for a packed batch -> dict of row arrays (app, slot, node, cpu, mem, gpu); with subtract the
        device-resident snapshot is charged with every reserved pod.  placed = (driver_node, executor_nodes, off)."""
        q = len(apps["count"])
        count = _np(apps["count"], np.int32)
        driver, execn, off = placed
        driver = _np(driver, np.int32); execn = _np(execn, np.int32)
        rows = int(((driver >= 0) * (1 + np.maximum(count, 0).astype(np.int64))).sum()) if q else 0
        t = {k: np.zeros(max(rows, 1), np.int32) for k in ("app", "slot", "node")}
        t.update({k: np.zeros(max(rows, 1), np.int64) for k in ("cpu", "mem", "gpu")})
        a = _apps(apps, off)
        r = gp_results(driver_node=_p(driver), executor_nodes=_p(execn), executor_nodes_cap=len(execn))
        tab = gp_reservation_table(rows_cap=len(t["app"]), app=_p(t["app"]), slot=_p(t["slot"]), node=_p(t["node"]),
                                   cpu_milli=_p(t["cpu"]), mem_bytes=_p(t["mem"]), gpu=_p(t["gpu"]), n_rows=0)
        self._check(load().gp_reserve_placements(self._h, C.byref(a), C.byref(r), 1 if subtract else 0, C.byref(tab)))
        return {k: v[:tab.n_rows] for k, v in t.items()}

    def apply_usage_delta(self, node, cpu, mem, gpu=None, sign=1):
        n, c, m, g = _np(node, np.int32), _np(cpu, np.int64), _np(mem, np.int64), _np(gpu, np.int64)
        self._check(load().gp_apply_usage_delta(self._h, len(n), _p(n), _p(c), _p(m), _p(g), sign))

    def packing_efficiency(self, apps: dict, placed, algo: int, charged: int = MODE_INDEPENDENT) -> np.ndarray:
        """computeAvgPackingEfficiencyForResult of each placed application over EVERY node of the snapshot, exactly summed
        -> (n_apps, 4) float64 {CPU, Memory, GPU, Max}.  placed = (driver_node, executor_nodes, off) as pack_batch returns
        them (zone results: (driver_node, executor_nodes, off) of the zone call).  algo decides what counts as reserved
        (MINIMAL_FRAGMENTATION: the driver only); charged = MODE_FIFO_* adds that one application's charged usage back first."""
        q = len(apps["count"])
        driver, execn, off = placed
        driver = _np(driver, np.int32); execn = _np(execn, np.int32)
        if execn is None or len(execn) == 0:
            execn = np.zeros(1, np.int32)
        avg = np.zeros((max(q, 1), 4), np.float64)
        a = _apps(apps, off)
        r = gp_results(driver_node=_p(driver), executor_nodes=_p(execn), executor_nodes_cap=len(execn))
        self._check(load().gp_packing_efficiency(self._h, C.byref(a), algo, C.byref(r), charged, _p(avg)))
        return avg[:q]

    def packing_efficiency_groups(self, apps: dict, placed, algo: int, instance_group, n_instance_groups: int,
                                  charged: int = MODE_INDEPENDENT) -> np.ndarray:
        """packing_efficiency with row i averaged over the nodes v with instance_group[v] == apps["group"][i] (absent: 0)
        instead of every node of the snapshot -- the reference's metric over the driver's instance group.  The FIFO charged
        modes allow at most one row per instance group; a placed node outside its row's instance group is refused.
        -> (n_apps, 4) float64 {CPU, Memory, GPU, Max}."""
        q = len(apps["count"])
        driver, execn, off = placed
        driver = _np(driver, np.int32); execn = _np(execn, np.int32)
        if execn is None or len(execn) == 0:
            execn = np.zeros(1, np.int32)
        ig = _np(instance_group, np.int32)
        avg = np.zeros((max(q, 1), 4), np.float64)
        a = _apps(apps, off, group=apps.get("group"))
        r = gp_results(driver_node=_p(driver), executor_nodes=_p(execn), executor_nodes_cap=len(execn))
        self._check(load().gp_packing_efficiency_groups(self._h, C.byref(a), algo, C.byref(r), charged, _p(ig),
                                                        int(n_instance_groups), _p(avg)))
        return avg[:q]

    def placement_metrics(self, apps: dict, placed, metric_zone, instance_group=None, n_instance_groups: int = 1,
                          n_metric_zones=None) -> np.ndarray:
        """What selectDriverNode reports about each placed application besides its packing efficiency: driver-executor
        collocation, executor node count and cross-zone pod pairs -> a PLACEMENT_DTYPE array of n_apps records.
        apps: count, [group], [off]; placed = (driver_node, executor_nodes, off) as pack_batch returns them; metric_zone: the
        interned failure-domain.beta.kubernetes.io/zone of each node (a missing label interned as "unknown-zone");
        instance_group: each node's instance group, -1 = none (None: every node is in every row's scope); n_metric_zones
        defaults to max(metric_zone) + 1."""
        q = len(apps["count"])
        driver, execn, off = placed
        driver = _np(driver, np.int32); execn = _np(execn, np.int32)
        if execn is None or len(execn) == 0:
            execn = np.zeros(1, np.int32)
        zone, ig = _np(metric_zone, np.int32), _np(instance_group, np.int32)
        out = np.zeros(max(q, 1), PLACEMENT_DTYPE)
        a = _apps(apps, off, group=apps.get("group"))
        r = gp_results(driver_node=_p(driver), executor_nodes=_p(execn), executor_nodes_cap=len(execn))
        if n_metric_zones is None:
            n_metric_zones = int(zone.max()) + 1 if len(zone) else 0
        self._check(load().gp_placement_metrics(self._h, C.byref(a), C.byref(r), len(zone), _p(zone), int(n_metric_zones), _p(ig),
                                                 int(n_instance_groups), _p(out)))
        return out[:q]

    def exceeds_cluster_capacity(self, alloc, apps: dict, packer: int, overhead=None, zone_id=None, n_zones=1, node_group=None,
                                 n_groups=1) -> np.ndarray:
        """DoesPodExceedClusterCapacity for a batch of stale drivers under one `binpack:` packer (BP_*), in one device call.
        alloc / overhead: (cpu, mem, gpu-or-None) per node; zone_id: interned ZoneLabel (None = one zone); node_group: affinity
        class per node, -1 = none (None = all 0).  apps: drv_*, exe_*, count and group (the driver's class, -1 = every node).
        -> uint8[n_apps], 1 = exceeds cluster capacity.  Leaves the context's snapshot and statistics untouched."""
        q = len(apps["count"])
        nd = _capacity_nodes(alloc, overhead, zone_id, n_zones, node_group, n_groups)
        a = _apps(apps, None, group=apps.get("group"))
        out = np.full(max(q, 1), 255, np.uint8)
        self._check(load().gp_exceeds_cluster_capacity(self._h, C.byref(nd), C.byref(a), int(packer), _p(out)))
        return out[:q]

    def exceeds_cluster_capacity_resident(self, alloc, overhead_node_id, apps: dict, packer: int, zone_id=None, n_zones=1,
                                          node_group=None, n_groups=1) -> np.ndarray:
        """exceeds_cluster_capacity with GetNonSchedulableOverhead from the resident overhead table
        (gp_exceeds_cluster_capacity_resident): overhead_node_id[n] = each node's overhead-table id (distinct, -1 = no records).
        Returns what exceeds_cluster_capacity returns with overhead = overhead_table_query(overhead_node_id)'s nonsched."""
        q = len(apps["count"])
        nd = _capacity_nodes(alloc, None, zone_id, n_zones, node_group, n_groups)
        oid = _np(overhead_node_id, np.int32)
        a = _apps(apps, None, group=apps.get("group"))
        out = np.full(max(q, 1), 255, np.uint8)
        self._check(load().gp_exceeds_cluster_capacity_resident(self._h, C.byref(nd), _p(oid), C.byref(a), int(packer), _p(out)))
        return out[:q]

    def match_node_affinity(self, enc: dict):
        """GetRequiredNodeAffinity(...).Match for every (affinity, node) of an affinity.encode() result, in one device call
        (gp_match_node_affinity).  -> (member uint32[n_aff][ceil(n / 32)], n_match int32[n_aff], n_error int32[n_aff]);
        a non-zero n_error is ListWithPredicate's error (the Predicate's failureInternal)."""
        lab, aff = _affinity_input(enc)
        return self._match(load().gp_match_node_affinity, lab, aff, lab.n_nodes)

    def match_node_affinity_resident(self, node_id, enc: dict):
        """match_node_affinity with the labels read in place from the label table (gp_match_node_affinity_resident): node_id
        [n] the label-table id of each node (-1 = no labels), enc the programs of LabelTable.encode_affinities()."""
        rl = _resident_labels(node_id)
        aff = _programs(enc)
        return self._match(load().gp_match_node_affinity_resident, rl, aff, rl.n_nodes)

    def _match(self, fn, lab, aff, n):
        words = (n + 31) // 32
        member = np.zeros((max(aff.n_aff, 1), max(words, 1)), np.uint32)
        n_match = np.zeros(max(aff.n_aff, 1), np.int32)
        n_error = np.zeros(max(aff.n_aff, 1), np.int32)
        out = gp_affinity_match(member=_p(member), n_match=_p(n_match), n_error=_p(n_error))
        self._check(fn(self._h, C.byref(lab), C.byref(aff), C.byref(out)))
        return member[:aff.n_aff, :words], n_match[:aff.n_aff], n_error[:aff.n_aff]

    def exceeds_cluster_capacity_affinity(self, alloc, enc: dict, apps: dict, packer: int, overhead=None, zone_id=None, n_zones=1):
        """exceeds_cluster_capacity with each driver's node set = the nodes its required affinity matches
        (gp_exceeds_cluster_capacity_affinity): enc from affinity.encode(); apps["group"] = the driver's affinity id.
        -> (exceeds uint8[n_apps], affinity_error uint8[n_apps]); exceeds[i] is undefined where affinity_error[i] = 1."""
        q = len(apps["count"])
        nd = _capacity_nodes(alloc, overhead, zone_id, n_zones, None, 0)
        lab, aff = _affinity_input(enc)
        a = _apps(apps, None, group=apps.get("group"))
        out = np.full(max(q, 1), 255, np.uint8)
        err = np.full(max(q, 1), 255, np.uint8)
        self._check(load().gp_exceeds_cluster_capacity_affinity(self._h, C.byref(nd), C.byref(lab), C.byref(aff), C.byref(a),
                                                                int(packer), _p(out), _p(err)))
        return out[:q], err[:q]

    def exceeds_cluster_capacity_affinity_resident(self, alloc, overhead_node_id, enc: dict, apps: dict, packer: int, zone_id=None,
                                                   n_zones=1):
        """exceeds_cluster_capacity_affinity with GetNonSchedulableOverhead from the resident overhead table
        (gp_exceeds_cluster_capacity_affinity_resident), overhead_node_id as in exceeds_cluster_capacity_resident."""
        q = len(apps["count"])
        nd = _capacity_nodes(alloc, None, zone_id, n_zones, None, 0)
        oid = _np(overhead_node_id, np.int32)
        lab, aff = _affinity_input(enc)
        a = _apps(apps, None, group=apps.get("group"))
        out = np.full(max(q, 1), 255, np.uint8)
        err = np.full(max(q, 1), 255, np.uint8)
        self._check(load().gp_exceeds_cluster_capacity_affinity_resident(self._h, C.byref(nd), _p(oid), C.byref(lab), C.byref(aff),
                                                                         C.byref(a), int(packer), _p(out), _p(err)))
        return out[:q], err[:q]

    def exceeds_cluster_capacity_affinity_label_table(self, alloc, overhead_node_id, node_id, enc: dict, apps: dict, packer: int,
                                                      zone_id=None, n_zones=1):
        """exceeds_cluster_capacity_affinity_resident with the labels read in place from the label table
        (gp_exceeds_cluster_capacity_affinity_label_table): node_id and enc as in match_node_affinity_resident."""
        q = len(apps["count"])
        nd = _capacity_nodes(alloc, None, zone_id, n_zones, None, 0)
        oid = _np(overhead_node_id, np.int32)
        rl = _resident_labels(node_id)
        aff = _programs(enc)
        a = _apps(apps, None, group=apps.get("group"))
        out = np.full(max(q, 1), 255, np.uint8)
        err = np.full(max(q, 1), 255, np.uint8)
        self._check(load().gp_exceeds_cluster_capacity_affinity_label_table(self._h, C.byref(nd), _p(oid), C.byref(rl), C.byref(aff),
                                                                            C.byref(a), int(packer), _p(out), _p(err)))
        return out[:q], err[:q]

    def reconcile_find_nodes(self, alloc, overhead, res_node, res, node_group, creation, apps: dict, n_groups: int,
                             unschedulable=None, ready=None, exec_cap=None, want_avail=True):
        """The failover reconciler's findNodes loop for a batch of stale drivers in one device call (gp_reconcile_find_nodes).
        alloc / overhead / res: (cpu, mem, gpu-or-None) triples (overhead may be None); res_node: node index per reservation row
        (hard and soft alike, -1 = unknown node); node_group: interned instanceGroupLabel per node; creation: int64 per node
        (UnixNano); apps: exe_cpu, exe_mem, exe_gpu (optional), count = max(0, Min - running) and group, in call order.
        -> (placed[q] (-1 = instance group not found), executor_nodes (CSR by off), off[q + 1], (cpu, mem, gpu) availability after
        the loop or None).  Leaves the context's snapshot and statistics untouched."""
        return self._reconcile(load().gp_reconcile_find_nodes, _usage_input(alloc, overhead, res_node, res), node_group, creation,
                               apps, n_groups, unschedulable, ready, exec_cap, want_avail)

    def reconcile_find_nodes_resident(self, node_id, alloc, overhead, node_group, creation, apps: dict, n_groups: int,
                                      unschedulable=None, ready=None, exec_cap=None, want_avail=True, overhead_node_id=None):
        """reconcile_find_nodes with the reservations from the resident reservation table (gp_reconcile_find_nodes_resident):
        node_id, overhead and overhead_node_id as in reschedule_from_reservations_resident.  Returns what reconcile_find_nodes
        returns on the equivalent rows, and leaves the context as it would."""
        return self._reconcile(load().gp_reconcile_find_nodes_resident, _resident_usage(node_id, alloc, overhead, overhead_node_id),
                               node_group, creation, apps, n_groups, unschedulable, ready, exec_cap, want_avail)

    def _reconcile(self, fn, ui, node_group, creation, apps, n_groups, unschedulable, ready, exec_cap, want_avail):
        n = ui.n_nodes
        ng, cr = _np(node_group, np.int32), _np(creation, np.int64)
        fu, fr = _np(unschedulable, np.uint8), _np(ready, np.uint8)
        nd = gp_reconcile_nodes(n_groups=int(n_groups), node_group=_p(ng), creation=_p(cr), unschedulable=_p(fu), ready=_p(fr))
        count = _np(apps["count"], np.int32)
        q = len(count)
        off = np.zeros(q + 1, np.int64)
        np.cumsum(count, out=off[1:])
        a = _apps(apps, off, group=apps.get("group"))
        placed = np.full(max(q, 1), -9, np.int32)
        cap = int(off[q]) if exec_cap is None else int(exec_cap)
        execn = np.full(max(cap, 1), -9, np.int32)
        av = [np.empty(max(n, 1), np.int64) for _ in range(3)] if want_avail else [None] * 3
        r = gp_reconcile_results(placed=_p(placed), executor_nodes=_p(execn), executor_nodes_cap=cap,
                                 avail_cpu_milli=_p(av[0]), avail_mem_bytes=_p(av[1]), avail_gpu=_p(av[2]))
        self._check(fn(self._h, C.byref(ui), C.byref(nd), C.byref(a), C.byref(r)))
        return placed[:q], execn[:int(off[q])], off, (tuple(x[:n] for x in av) if want_avail else None)

    def node_overhead(self, enc: dict):
        """GetOverhead and GetNonSchedulableOverhead for the listed nodes in one device call (gp_node_overhead), over an
        overhead.encode() result (or the same keys given by hand; a missing optional column is NULL).
        -> (overhead (cpu, mem, gpu), nonsched (cpu, mem, gpu), has_reservation uint8[n_pods], n_warned): the triples in
        enc["node_ids"] order, as build_availability, prepare_cluster, exceeds_cluster_capacity and reconcile_find_nodes
        take them.  Leaves the context's snapshot and statistics untouched."""
        col = {k: _np(enc.get(k), t) for k, t in _OVERHEAD_COLS.items()}
        n_pods = int(enc["n_pods"]) if "n_pods" in enc else len(col["node_id"])
        pods = gp_overhead_pods(n_pods=n_pods, n_node_ids=int(enc["n_node_ids"]), n_app_keys=int(enc["n_app_keys"]),
                                n_app_ids=int(enc["n_app_ids"]), n_names=int(enc["n_names"]),
                                **{k: _p(col[k]) for k in _OVERHEAD_COLS if k in gp_overhead_pods.__dict__})
        rsv = gp_overhead_reservations(n_rr=int(enc["n_rr"]) if "n_rr" in enc else len(col["rr_app_key"]),
                                       n_soft=int(enc["n_soft"]) if "n_soft" in enc else len(col["soft_app_id"]),
                                       **{k: _p(col[k]) for k in _OVERHEAD_COLS if k in gp_overhead_reservations.__dict__})
        qn = col["node_ids"]
        n = 0 if qn is None else len(qn)
        res = [np.zeros(max(n, 1), np.int64) for _ in range(6)]
        has = np.zeros(max(n_pods, 1), np.uint8)
        warned = C.c_int64(-1)
        out = gp_overhead_out(*[_p(x) for x in res], _p(has), C.addressof(warned))
        self._check(load().gp_node_overhead(self._h, C.byref(pods), C.byref(rsv), n, _p(qn), C.byref(out)))
        return tuple(x[:n] for x in res[:3]), tuple(x[:n] for x in res[3:]), has[:n_pods], warned.value

    # ---- the resident overhead table (gp_overhead_table_*) ---------------------------------------------------------------
    def overhead_table_reset(self, n_slots, n_node_ids, n_app_keys, n_app_ids, n_names):
        """Replace the context's overhead table with an empty one of these capacities."""
        z = gp_overhead_table_size(int(n_slots), int(n_node_ids), int(n_app_keys), int(n_app_ids), int(n_names))
        # recorded once the library holds the new table: a refused reset keeps the table and size held before, and after a
        # reset that fails with a CUDA error every query is refused before anything is downloaded
        self._check(load().gp_overhead_table_reset(self._h, C.byref(z)))
        self._oht_slots = int(n_slots)

    def overhead_table_update(self, delta: dict):
        """One gp_overhead_table_update over the arrays of overhead.OverheadTable.delta() (or the same keys given by hand; a
        missing optional column is NULL; the "reset" entry is not read here)."""
        col = {k: _np(delta.get(k), t) for k, t in _DELTA_COLS.items()}
        n = lambda k: 0 if col[k] is None else len(col[k])
        d = gp_overhead_delta(n_write=int(delta.get("n_write", n("slot"))), n_rr=int(delta.get("n_rr", n("rr_app_key"))),
                              n_member=int(delta.get("n_member", n("member_kind"))), **{k: _p(v) for k, v in col.items()})
        self._check(load().gp_overhead_table_update(self._h, C.byref(d)))

    def overhead_table_query(self, node_ids, has_reservation=True):
        """The table's GetOverhead and GetNonSchedulableOverhead for the listed node ids -> the tuple of node_overhead, with
        has_reservation over every slot of the table (None when not asked for)."""
        qn = _np(node_ids, np.int32)
        n = len(qn)
        res = [np.zeros(max(n, 1), np.int64) for _ in range(6)]
        slots = getattr(self, "_oht_slots", 0)          # [n_slots] of the table held; before any reset the query is refused
        has = np.zeros(max(slots, 1), np.uint8) if has_reservation else None
        warned = C.c_int64(-1)
        out = gp_overhead_out(*[_p(x) for x in res], _p(has), C.addressof(warned))
        self._check(load().gp_overhead_table_query(self._h, n, _p(qn), C.byref(out)))
        return (tuple(x[:n] for x in res[:3]), tuple(x[:n] for x in res[3:]),
                None if has is None else has[:slots], warned.value)

    # ---- the resident reservation table (gp_reservation_table_*) ---------------------------------------------------------
    def reservation_table_reset(self, n_slots, n_node_ids):
        """Replace the context's reservation table with an empty one of these capacities."""
        self._check(load().gp_reservation_table_reset(self._h, C.byref(gp_reservation_table_size(int(n_slots), int(n_node_ids)))))

    def reservation_table_update(self, delta: dict):
        """One gp_reservation_table_update over the arrays of reservations.ReservationTable.delta() (slot, node_id, cpu_milli,
        mem_bytes and optionally gpu; the "reset" entry is not read here)."""
        col = {k: _np(delta.get(k), t) for k, t in _RT_DELTA_COLS.items()}
        d = gp_reservation_delta(n_write=0 if col["slot"] is None else len(col["slot"]), **{k: _p(v) for k, v in col.items()})
        self._check(load().gp_reservation_table_update(self._h, C.byref(d)))

    # ---- the resident label table (gp_label_table_*) ---------------------------------------------------------------------
    def label_table_reset(self, n_node_ids, max_labels, n_keys, n_values):
        """Replace the context's label table with an empty one of these capacities."""
        z = gp_label_table_size(int(n_node_ids), int(max_labels), int(n_keys), int(n_values))
        self._check(load().gp_label_table_reset(self._h, C.byref(z)))

    def label_table_update(self, delta: dict):
        """One gp_label_table_update over the arrays of affinity.LabelTable.delta() (row_node, row_off, label_key, label_val,
        value_id, value_int_ok, value_int; a missing column is NULL; the "reset" entry is not read here)."""
        col = {k: _np(delta.get(k), t) for k, t in _LT_DELTA_COLS.items()}
        n = lambda k: 0 if col[k] is None else len(col[k])
        d = gp_label_delta(n_rows=int(delta.get("n_rows", n("row_node"))), n_values=int(delta.get("n_values", n("value_id"))),
                           **{k: _p(v) for k, v in col.items()})
        self._check(load().gp_label_table_update(self._h, C.byref(d)))

    # ---- the resident node table (gp_node_table_*) and the node-table Predicate entries ----------------------------------
    def node_table_reset(self, n_node_ids):
        """Replace the context's node table with an empty one of this capacity."""
        self._check(load().gp_node_table_reset(self._h, C.byref(gp_node_table_size(int(n_node_ids), 0))))

    def node_table_update(self, delta: dict):
        """One gp_node_table_update over the arrays of nodes.NodeTable.delta() (node_id, present, alloc_cpu_milli,
        alloc_mem_bytes, alloc_gpu, unschedulable, ready, name_key, creation; a missing column is NULL; "reset" is not read
        here)."""
        col = {k: _np(delta.get(k), t) for k, t in _NT_DELTA_COLS.items()}
        d = gp_node_delta(n_write=0 if col["node_id"] is None else len(col["node_id"]), **{k: _p(v) for k, v in col.items()})
        self._check(load().gp_node_table_update(self._h, C.byref(d)))

    def prepare_cluster_groups_node_table(self, nodes: dict, instance_group, n_instance_groups, orders=True):
        """prepare_cluster_groups_resident with the node columns from the node and label tables: nodes holds the keyword
        arguments of the gp_node_table_nodes (node_table_id, reservation_id, overhead_node_id, is_driver_candidate, zone_key,
        zone_value, n_zones, zone_missing, instance_group_key, instance_group_value, driver_rank_key, driver_rank_value,
        executor_rank_key, executor_rank_value, zone_id_out, instance_group_out).  instance_group: an array, or None to take
        the instance groups from the labels (or every node in 0 without instance_group_key).  Returns what
        prepare_cluster_groups_resident returns on the equivalent columns."""
        nt = _node_table_nodes(**nodes)
        return self._prepare_groups(_node_table_entry(load().gp_prepare_cluster_groups_node_table), nt, instance_group,
                                    n_instance_groups, None, int(nt.n_zones), None, None, None, None, None, None, orders)

    def prepare_cluster_zones_groups_node_table(self, nodes: dict, instance_group, n_instance_groups, kind=LAYOUT_AZ_AWARE, layout=True):
        """prepare_cluster_zones_groups_resident with the node columns from the node and label tables (nodes and
        instance_group as in prepare_cluster_groups_node_table)."""
        nt = _node_table_nodes(**nodes)
        return self._prepare_zones_groups(_node_table_entry(load().gp_prepare_cluster_zones_groups_node_table), nt, instance_group,
                                          n_instance_groups, None, int(nt.n_zones), None, None, None, None, None, None, kind, layout)

    def reschedule_from_reservations_node_table(self, nodes: dict, exe, min_frag=False, hosting=None, keep_topology_zone=None,
                                                topology_zone=None):
        """reschedule_from_reservations_resident with the node columns from the node and label tables (nodes as in
        prepare_cluster_groups_node_table; instance groups do not apply)."""
        nt = _node_table_nodes(**nodes)
        return self._reschedule(_node_table_entry(load().gp_reschedule_from_reservations_node_table), nt, exe, min_frag, hosting,
                                None, int(nt.n_zones), None, None, None, None, keep_topology_zone, topology_zone)

    def reconcile_find_nodes_node_table(self, nodes: dict, apps: dict, n_groups: int, instance_group_missing: int, exec_cap=None,
                                        want_avail=True):
        """reconcile_find_nodes_resident with the node columns from the node and label tables
        (gp_reconcile_find_nodes_node_table): nodes as in prepare_cluster_groups_node_table (is_driver_candidate and the rank
        keys ignored); the instance group of a node is the index of its instance_group_key value in instance_group_value, a
        node without the label is in instance_group_missing (the group of ""), and every node in 0 without instance_group_key.
        Returns what reconcile_find_nodes_resident returns on the equivalent columns."""
        if int(nodes.get("instance_group_key", -1)) >= 0 and len(nodes.get("instance_group_value", ())) != int(n_groups):
            raise ValueError("instance_group_value must list exactly n_groups value ids (the call reads n_groups of them)")
        nt = _node_table_nodes(**nodes)

        def fn(h, nt_ref, nd_ref, *rest):
            return load().gp_reconcile_find_nodes_node_table(h, nt_ref, int(n_groups), int(instance_group_missing), *rest)
        return self._reconcile(fn, nt, None, None, apps, n_groups, None, None, exec_cap, want_avail)

    def exceeds_cluster_capacity_node_table(self, nodes: dict, apps: dict, packer: int, node_group=None, n_groups=1) -> np.ndarray:
        """exceeds_cluster_capacity_resident with allocatable from the node table, zone_id from the label table and
        overhead_node_id from nodes (gp_exceeds_cluster_capacity_node_table); reservation_id may be omitted."""
        q = len(apps["count"])
        nt = _node_table_nodes(**dict({"reservation_id": None}, **nodes))
        grp = _np(node_group, np.int32)
        a = _apps(apps, None, group=apps.get("group"))
        out = np.full(max(q, 1), 255, np.uint8)
        self._check(load().gp_exceeds_cluster_capacity_node_table(self._h, C.byref(nt), _p(grp), int(n_groups), C.byref(a), int(packer),
                                                                  _p(out)))
        return out[:q]

    def exceeds_cluster_capacity_affinity_node_table(self, nodes: dict, enc: dict, apps: dict, packer: int):
        """exceeds_cluster_capacity_affinity_label_table with allocatable, zone_id and the label rows from nodes
        (gp_exceeds_cluster_capacity_affinity_node_table); enc as in match_node_affinity_resident."""
        q = len(apps["count"])
        nt = _node_table_nodes(**dict({"reservation_id": None}, **nodes))
        aff = _programs(enc)
        a = _apps(apps, None, group=apps.get("group"))
        out = np.full(max(q, 1), 255, np.uint8)
        err = np.full(max(q, 1), 255, np.uint8)
        self._check(load().gp_exceeds_cluster_capacity_affinity_node_table(self._h, C.byref(nt), C.byref(aff), C.byref(a), int(packer),
                                                                           _p(out), _p(err)))
        return out[:q], err[:q]

    # ---- the resident driver table (gp_driver_table_*) and the driver-table FIFO entries ----------------------------------
    def driver_table_reset(self, n_slots, n_groups, n_schedulers):
        """Replace the context's driver table with an empty one of these capacities."""
        self._check(load().gp_driver_table_reset(self._h, C.byref(gp_driver_table_size(int(n_slots), int(n_groups), int(n_schedulers), 0))))

    def driver_table_update(self, delta: dict):
        """One gp_driver_table_update over the arrays of drivers.DriverTable.delta() (slot, present, creation, scheduler, group,
        the six quantity columns, min_executor_count, exact; a missing column is NULL; "reset" is not read here)."""
        col = {k: _np(delta.get(k), t) for k, t in _DT_DELTA_COLS.items()}
        d = gp_driver_delta(n_write=0 if col["slot"] is None else len(col["slot"]), **{k: _p(v) for k, v in col.items()})
        self._check(load().gp_driver_table_update(self._h, C.byref(d)))

    def _driver_queue(self, queue: dict, queue_cap):
        """gp_driver_queue over queue = dict(requesting_slot=-1, scheduler=0, predicate_group=0, snapshot_group=None,
        enforce_after_ns=None, now=0) with out arrays for queue_cap entries; -> (struct, outs dict)"""
        sg, age = _np(queue.get("snapshot_group"), np.int32), _np(queue.get("enforce_after_ns"), np.int64)
        outs = dict(queue_slot=np.empty(max(queue_cap, 1), np.int32), off=np.empty(queue_cap + 1, np.int64),
                    n_queued=C.c_int32(-9), n_executors=C.c_int64(-9), ties=C.c_int32(-9))
        dq = gp_driver_queue(requesting_slot=int(queue.get("requesting_slot", -1)), scheduler=int(queue.get("scheduler", 0)),
                             predicate_group=int(queue.get("predicate_group", 0)), queue_cap=int(queue_cap), snapshot_group=_p(sg),
                             enforce_after_ns=_p(age), now_unix_nano=int(queue.get("now", 0)), queue_slot=_p(outs["queue_slot"]),
                             exec_out_off=_p(outs["off"]), n_queued=C.addressof(outs["n_queued"]),
                             n_executors=C.addressof(outs["n_executors"]), undefined_ties=C.addressof(outs["ties"]))
        dq._keep = (sg, age, outs)
        return dq, outs

    def _driver_table_call(self, queue, queue_cap, exec_cap, retry, call):
        """call(gp_driver_queue, outs, exec_cap) -> status.  Default capacities: the table's slots + 1 and 4 executors per
        entry; with retry, a GP_ERR_CAPACITY is retried once with the sizes the call wrote back."""
        if queue_cap is None:
            queue_cap = int(queue.get("n_slots", 0)) + 1
        if exec_cap is None:
            exec_cap = 4 * queue_cap
        dq, outs = self._driver_queue(queue, queue_cap)
        st = call(dq, outs, exec_cap)
        if st == 5 and retry:
            queue_cap = max(queue_cap, outs["n_queued"].value)
            exec_cap = max(exec_cap, int(outs["n_executors"].value))
            dq, outs = self._driver_queue(queue, queue_cap)
            st = call(dq, outs, exec_cap)
        self._check(st)
        n = outs["n_queued"].value
        return dict(queue_slot=outs["queue_slot"][:n].copy(), off=outs["off"][:n + 1].copy(), n_queued=n,
                    n_executors=outs["n_executors"].value, undefined_ties=outs["ties"].value)

    def pack_fifo_driver_table(self, queue: dict, algo: int, mode: int, queue_cap=None, exec_cap=None, retry=True) -> dict:
        """gp_pack_fifo_driver_table: the FIFO queue selected and ordered from the driver table (queue as in _driver_queue,
        plus n_slots for the default capacity), packed over the held snapshot.  -> dict with queue_slot, off, n_queued,
        n_executors, undefined_ties, driver_node and executor_nodes."""
        res = {}

        def call(dq, outs, cap):
            res["drv"] = np.empty(max(dq.queue_cap, 1), np.int32)
            res["exe"] = np.empty(max(cap, 1), np.int32)      # defined for placed drivers only, as gp_results says
            r = gp_results(driver_node=_p(res["drv"]), executor_nodes=_p(res["exe"]), executor_nodes_cap=int(cap))
            return load().gp_pack_fifo_driver_table(self._h, C.byref(dq), int(algo), int(mode), C.byref(r))
        out = self._driver_table_call(queue, queue_cap, exec_cap, retry, call)
        out["driver_node"] = res["drv"][:out["n_queued"]].copy()
        out["executor_nodes"] = res["exe"][:out["n_executors"]].copy()
        return out

    def pack_fifo_zones_groups_driver_table(self, queue: dict, packer: int, mode: int, queue_cap=None, exec_cap=None, retry=True) -> dict:
        """gp_pack_fifo_zones_groups_driver_table over the layout prepare_cluster_zones_groups left: -> the dict of
        pack_fifo_driver_table plus zone and avg_efficiency."""
        res = {}

        def call(dq, outs, cap):
            q = max(dq.queue_cap, 1)
            res.update(zone=np.empty(q, np.int32), drv=np.empty(q, np.int32), exe=np.empty(max(cap, 1), np.int32),
                       avg=np.zeros((q, 4), np.float64))
            r = gp_zone_results(zone=_p(res["zone"]), driver_node=_p(res["drv"]), executor_nodes=_p(res["exe"]), executor_nodes_cap=int(cap),
                                avg_efficiency=_p(res["avg"]))
            return load().gp_pack_fifo_zones_groups_driver_table(self._h, C.byref(dq), int(packer), int(mode), None, C.byref(r))
        out = self._driver_table_call(queue, queue_cap, exec_cap, retry, call)
        n = out["n_queued"]
        out.update(zone=res["zone"][:n].copy(), driver_node=res["drv"][:n].copy(), executor_nodes=res["exe"][:out["n_executors"]].copy(),
                   avg_efficiency=res["avg"][:n].copy())
        return out

    def exceeds_cluster_capacity_driver_table(self, nodes: dict, enc: dict, scheduler: int, timeout_ns: int, now: int, packer: int,
                                              cap=None, retry=True) -> dict:
        """gp_exceeds_cluster_capacity_driver_table: the marker's sweep over the driver table's stale rows (scheduler id,
        creation + timeout_ns < now), nodes as in exceeds_cluster_capacity_affinity_node_table and enc the programs the
        table's affinity ids index (drivers.DriverTable.affinity_programs encoded).  cap defaults to 64; with retry a
        GP_ERR_CAPACITY is retried once with the size the call wrote back.  -> dict with stale_slot, exceeds and
        outcome (0 answered, 1 affinity error, 2 outside the model) in (creation, slot) order."""
        nt = _node_table_nodes(**dict({"reservation_id": None}, **nodes))
        aff = _programs(enc)
        cap = 64 if cap is None else int(cap)

        def call(cap):
            o = dict(slot=np.full(max(cap, 1), -9, np.int32), exceeds=np.full(max(cap, 1), 255, np.uint8),
                     outcome=np.full(max(cap, 1), 255, np.uint8), n=C.c_int32(-9))
            sw = gp_stale_sweep(scheduler=int(scheduler), cap=int(cap), timeout_ns=int(timeout_ns), now_unix_nano=int(now),
                                stale_slot=_p(o["slot"]), exceeds=_p(o["exceeds"]), outcome=_p(o["outcome"]), n_stale=C.addressof(o["n"]))
            return load().gp_exceeds_cluster_capacity_driver_table(self._h, C.byref(nt), C.byref(aff), C.byref(sw), int(packer)), o
        st, o = call(cap)
        if st == 5 and retry:
            st, o = call(max(cap, o["n"].value))
        self._check(st)
        n = o["n"].value
        return dict(stale_slot=o["slot"][:n].copy(), exceeds=o["exceeds"][:n].copy(), outcome=o["outcome"][:n].copy())

    # ---- bound calls: what a shim does -- marshal the argument structs ONCE over its long-lived buffers, then one FFI call
    # per Predicate (the numpy / ctypes marshalling of set_snapshot() / pack_batch() costs more than a small batch's kernels)
    def bind_snapshot(self, avail_cpu, avail_mem, avail_gpu, exec_order, drv_order, exec_off, drv_off):
        """-> zero-argument callable running gp_set_snapshot on these (caller-owned, stable) arrays."""
        keep = [_np(avail_cpu, np.int64), _np(avail_mem, np.int64), _np(avail_gpu, np.int64), _np(exec_order, np.int32),
                _np(drv_order, np.int32), _np(exec_off, np.int32), _np(drv_off, np.int32)]
        n = gp_nodes(n_nodes=len(keep[0]), avail_cpu_milli=_p(keep[0]), avail_mem_bytes=_p(keep[1]), avail_gpu=_p(keep[2]),
                     n_groups=len(keep[5]) - 1, exec_off=_p(keep[5]), exec_order=_p(keep[3]), drv_off=_p(keep[6]), drv_order=_p(keep[4]))
        fn, h, ref = load().gp_set_snapshot, self._h, C.byref(n)
        self.n_nodes = len(keep[0])

        def call(_keep=(keep, n)):
            st = fn(h, ref)
            if st != 0:
                self._check(st)
        return call

    def bind_batch(self, apps: dict, algo: int, mode: int, out, wire: dict):
        """-> zero-argument callable running gp_pack_batch_wire on these (caller-owned, stable) arrays; results land in `out`."""
        bits = int(wire.get("quantity_bits", 64))
        qdt = np.int64 if bits == 64 else np.int32
        q = len(apps["count"])
        keep = {k: _np(apps.get(k), qdt) for k in ("drv_cpu", "drv_mem", "drv_gpu", "exe_cpu", "exe_mem", "exe_gpu")}
        keep["count"] = _np(apps["count"], np.int32)
        keep["group"] = _np(apps.get("group"), np.int32)
        keep["young"] = _np(apps.get("young"), np.uint8)
        keep["off"] = _np(apps.get("off"), np.int64) if wire.get("offsets", True) else None
        if wire.get("offsets", True) and keep["off"] is None:
            raise ValueError("bind_batch: wire.offsets is set but apps has no 'off'")
        driver_node, executor_nodes = out
        a = gp_apps_wire(n_apps=q, quantity_bits=bits, mem_shift=int(wire.get("mem_shift", 0)),
                         drv_cpu=_p(keep["drv_cpu"]), drv_mem=_p(keep["drv_mem"]), drv_gpu=_p(keep["drv_gpu"]),
                         exe_cpu=_p(keep["exe_cpu"]), exe_mem=_p(keep["exe_mem"]), exe_gpu=_p(keep["exe_gpu"]),
                         exe_count=_p(keep["count"]), group=_p(keep["group"]), skip_if_no_fit=_p(keep["young"]),
                         exec_out_off=_p(keep["off"]))
        r = gp_results_wire(driver_node=_p(driver_node), executor_nodes=_p(executor_nodes),
                            executor_nodes_cap=len(executor_nodes), node_bits=int(wire.get("node_bits", 32)))
        fn, h, ra, rr = load().gp_pack_batch_wire, self._h, C.byref(a), C.byref(r)

        def call(_keep=(keep, a, r, out)):
            st = fn(h, ra, algo, mode, rr)
            if st != 0:
                self._check(st)
        return call

    def pack_one(self, algo, drv, exe, count):
        """binpack.SparkBinPackFunction for one app -> (has_capacity, driver_node, executor_nodes)."""
        has = C.c_int32(0); d = C.c_int32(-1)
        en = np.full(max(count, 1), -9, np.int32)
        self._check(load().gp_pack_one(self._h, algo, int(drv[0]), int(drv[1]), int(drv[2]), int(exe[0]), int(exe[1]),
                                       int(exe[2]), int(count), C.byref(has), C.byref(d), _p(en)))
        return bool(has.value), d.value, en[:count] if has.value else en[:0]

    def stats(self) -> dict:
        """gp_last_stats of the last pack call.  scan_path_apps: independent tightly / evenly batches count the applications
        the node-order scan decided instead of the capacity tables; the FIFO modes count the applications the whole CTA
        decided instead of warp 0 alone (all evaluated ones with GANGPACK_FIFO_WARP=0); pack_fifo_az_aware and
        pack_batch_az_aware count the applications for which the undivided fallback ran."""
        s = gp_stats()
        self._check(load().gp_last_stats(self._h, C.byref(s)))
        return {"nodes_scanned": s.nodes_scanned, "drivers_tried": s.drivers_tried, "kernel_launches": s.kernel_launches,
                "pack_kernel_ns": s.pack_kernel_ns, "prep_kernel_ns": s.prep_kernel_ns,
                "scan_path_apps": s.scan_path_apps, "scan_path_nodes": s.scan_path_nodes}

    # ---- device-resident (torch tensors on this context's device) ----------------------------
    def stream_handle(self) -> int:
        return load().gp_stream(self._h) or 0

    def synchronize(self):
        self._check(load().gp_synchronize(self._h))

    def set_snapshot_device(self, cpu, mem, gpu, exec_off, exec_order, drv_off, drv_order, stream: int = 0):
        """All arguments are torch CUDA tensors (int64 / int32); kept alive by the caller."""
        n = gp_nodes(n_nodes=cpu.numel(), avail_cpu_milli=cpu.data_ptr(), avail_mem_bytes=mem.data_ptr(),
                     avail_gpu=gpu.data_ptr() if gpu is not None else None, n_groups=exec_off.numel() - 1,
                     exec_off=exec_off.data_ptr(), exec_order=exec_order.data_ptr(), drv_off=drv_off.data_ptr(),
                     drv_order=drv_order.data_ptr())
        self._check(load().gp_set_snapshot_device(self._h, C.byref(n), exec_order.numel(), drv_order.numel(),
                                                  stream or None))
        self.n_nodes = cpu.numel()

    def pack_batch_device(self, t: dict, algo: int, mode: int, driver_node, executor_nodes, stream: int = 0):
        """t: dict of torch CUDA tensors (drv_cpu, drv_mem, [drv_gpu], exe_cpu, exe_mem, [exe_gpu], count, [group],
        [young], off).  Asynchronous on `stream` (0 = the context's stream)."""
        def dp(name):
            v = t.get(name)
            return v.data_ptr() if v is not None else None
        a = gp_apps(n_apps=t["count"].numel(), drv_cpu_milli=dp("drv_cpu"), drv_mem_bytes=dp("drv_mem"),
                    drv_gpu=dp("drv_gpu"), exe_cpu_milli=dp("exe_cpu"), exe_mem_bytes=dp("exe_mem"),
                    exe_gpu=dp("exe_gpu"), exe_count=dp("count"), group=dp("group"), skip_if_no_fit=dp("young"),
                    exec_out_off=dp("off"))
        r = gp_results(driver_node=driver_node.data_ptr(), executor_nodes=executor_nodes.data_ptr(),
                       executor_nodes_cap=executor_nodes.numel())
        self._check(load().gp_pack_batch_device(self._h, C.byref(a), algo, mode, C.byref(r), stream or None))

    def placement_metrics_device(self, t: dict, driver_node, executor_nodes, metric_zone, out, n_metric_zones: int,
                                 instance_group=None, n_instance_groups: int = 1, status=None, stream: int = 0):
        """placement_metrics on torch CUDA tensors, e.g. pack_batch_device's inputs and outputs in place: t as there (count,
        [group], [off]), out a uint8 tensor of PLACEMENT_DTYPE.itemsize * n_apps bytes (view it with PLACEMENT_DTYPE), status an int32 tensor of one
        element receiving the call's status (0 = ok) once the work has run.  Asynchronous on `stream` (0 = the context's)."""
        def dp(v):
            return v.data_ptr() if v is not None else None
        a = gp_apps(n_apps=t["count"].numel(), exe_count=dp(t["count"]), group=dp(t.get("group")), exec_out_off=dp(t.get("off")))
        r = gp_results(driver_node=driver_node.data_ptr(), executor_nodes=executor_nodes.data_ptr(),
                       executor_nodes_cap=executor_nodes.numel())
        self._check(load().gp_placement_metrics_device(self._h, C.byref(a), C.byref(r), metric_zone.numel(), dp(metric_zone),
                                                        int(n_metric_zones), dp(instance_group), int(n_instance_groups), dp(out),
                                                        dp(status), stream or None))


class MultiGangPacker:
    """gp_multi: one host process, several GPUs (or several contexts on one GPU).  Same call shapes as GangPacker."""

    def __init__(self, devices):
        L = load()
        self._h = C.c_void_p()
        dev = np.ascontiguousarray(devices, dtype=np.int32)
        st = L.gp_multi_create(C.byref(self._h), dev.ctypes.data, len(dev))
        if st != 0:
            raise GangpackError(st, (L.gp_last_error(None) or b"").decode())
        self.n_devices = len(dev)
        self._pinned = []

    def close(self):
        if getattr(self, "_h", None):
            for ctx, ptr in self._pinned:
                load().gp_free_pinned(ctx, ptr)
            self._pinned = []
            load().gp_multi_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, st):
        if st != 0:
            raise GangpackError(st, (load().gp_multi_last_error(self._h) or b"").decode())

    def pinned(self, shape, dtype) -> np.ndarray:
        """Pinned host memory (portable: usable by every device of the handle)."""
        dt = np.dtype(dtype)
        n = int(np.prod(shape)) if np.ndim(shape) else int(shape)
        nbytes = max(n * dt.itemsize, 1)
        ptr = C.c_void_p()
        ctx = load().gp_multi_ctx(self._h, 0)
        st = load().gp_alloc_pinned(ctx, nbytes, C.byref(ptr))
        if st != 0:
            raise GangpackError(st, (load().gp_last_error(ctx) or b"").decode())
        self._pinned.append((ctx, ptr))
        buf = (C.c_char * nbytes).from_address(ptr.value)
        return np.frombuffer(buf, dtype=dt, count=n).reshape(shape)

    def set_snapshot(self, avail_cpu, avail_mem, avail_gpu, exec_order, drv_order, exec_off=None, drv_off=None):
        cpu, mem, gpu = _np(avail_cpu, np.int64), _np(avail_mem, np.int64), _np(avail_gpu, np.int64)
        eo, do = _np(exec_order, np.int32), _np(drv_order, np.int32)
        eoff = _np(exec_off if exec_off is not None else [0, len(eo)], np.int32)
        doff = _np(drv_off if drv_off is not None else [0, len(do)], np.int32)
        n = gp_nodes(n_nodes=len(cpu), avail_cpu_milli=_p(cpu), avail_mem_bytes=_p(mem), avail_gpu=_p(gpu),
                     n_groups=len(eoff) - 1, exec_off=_p(eoff), exec_order=_p(eo), drv_off=_p(doff), drv_order=_p(do))
        self._check(load().gp_multi_set_snapshot(self._h, C.byref(n)))
        self.n_nodes, self.n_groups = len(cpu), len(eoff) - 1

    def get_snapshot(self):
        cpu = np.empty(self.n_nodes, np.int64); mem = np.empty(self.n_nodes, np.int64); gpu = np.empty(self.n_nodes, np.int64)
        self._check(load().gp_multi_get_snapshot(self._h, _p(cpu), _p(mem), _p(gpu)))
        return cpu, mem, gpu

    def group_owner(self):
        o = np.empty(self.n_groups, np.int32)
        self._check(load().gp_multi_group_owner(self._h, _p(o)))
        return o

    def pack_batch(self, apps: dict, algo: int, mode: int = MODE_INDEPENDENT, out=None, wire=None):
        """Same contract as GangPacker.pack_batch (wire=None -> int64 quantities, offsets given, int32 node indices)."""
        wire = dict(wire or dict(quantity_bits=64, node_bits=32, offsets=True))
        q = len(apps["count"])
        count = _np(apps["count"], np.int32)
        off = _np(apps.get("off"), np.int64)
        derive = not wire.get("offsets", True)
        if off is None and not (derive and out is not None):      # hot path (caller's buffers, device-derived offsets): no host cumsum
            off = np.zeros(q + 1, np.int64)
            np.cumsum(np.maximum(count, 0), out=off[1:])
        bits = int(wire.get("quantity_bits", 64))
        qdt = np.int64 if bits == 64 else np.int32
        arrs = {k: _np(apps.get(k), qdt) for k in ("drv_cpu", "drv_mem", "drv_gpu", "exe_cpu", "exe_mem", "exe_gpu")}
        grp, young = _np(apps.get("group"), np.int32), _np(apps.get("young"), np.uint8)
        total = (int(off[-1]) if q else 0) if off is not None else len(out[1])
        node_bits = int(wire.get("node_bits", 32))
        if out is None:
            driver_node = np.full(q, -9, np.int32)
            executor_nodes = np.full(max(total, 1), -9 if node_bits == 32 else 65535, np.int32 if node_bits == 32 else np.uint16)
        else:
            driver_node, executor_nodes = out
        a = gp_apps_wire(n_apps=q, quantity_bits=bits, mem_shift=int(wire.get("mem_shift", 0)),
                         drv_cpu=_p(arrs["drv_cpu"]), drv_mem=_p(arrs["drv_mem"]), drv_gpu=_p(arrs["drv_gpu"]),
                         exe_cpu=_p(arrs["exe_cpu"]), exe_mem=_p(arrs["exe_mem"]), exe_gpu=_p(arrs["exe_gpu"]),
                         exe_count=_p(count), group=_p(grp), skip_if_no_fit=_p(young),
                         exec_out_off=None if derive else _p(off))
        r = gp_results_wire(driver_node=_p(driver_node), executor_nodes=_p(executor_nodes),
                            executor_nodes_cap=len(executor_nodes), node_bits=node_bits)
        self._check(load().gp_multi_pack_batch(self._h, C.byref(a), algo, mode, C.byref(r)))
        return driver_node, executor_nodes[:total], off
