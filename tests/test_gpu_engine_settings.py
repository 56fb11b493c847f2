"""The engine's run-time settings (DBEEL_* variables read at engine creation) choose which kernel instantiations a job runs and
how they are launched; every setting must give the same bytes.  Each spec below gets its own engine (one at a time), first
proves that it really runs the kernels it claims, then reruns the existing parity corpus on it -- the test functions of the
other files, called with the spec's engine -- and the persistent extract's step and wave borders, which nothing else
reaches.  A CPU test keeps the matrix complete: every DBEEL_* variable the native code reads is either a spec here or named
with the test that sets it."""
import hashlib
import inspect
import os
import re

import numpy as np
import pytest

import oracle
from dbeel_b200 import capi, sstable
from dbeel_b200 import workloads as W

import test_gpu_buffer_edges as edges
import test_gpu_cfg5 as cfg5_tests
import test_gpu_get_values as get_values
import test_gpu_get_values_stream as get_values_stream
import test_gpu_lookup as lookup
import test_gpu_merge_final as merge_final
import test_gpu_merge_final_pipeline as merge_final_pipeline
import test_gpu_parity as parity
import test_gpu_reader as reader
import test_gpu_reference_reader as reference_reader
import test_gpu_scan as scan
import test_gpu_scan_stream as scan_stream
import test_gpu_wal as wal
import test_host_tree as host_tree
import test_routing as routing
from helpers import BASE_TS, assert_run_equal, model_compact, model_flush, random_runs
from test_gpu_merge_final_pipeline import _engine
from test_gpu_parity import SEED, check_against_oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SPECS = {
    "default": {},
    "narrow0": {"DBEEL_NARROW": "0"},
    "narrow0-fused0": {"DBEEL_NARROW": "0", "DBEEL_FUSED_FINAL": "0"},
    "fused0": {"DBEEL_FUSED_FINAL": "0"},
    "persist0": {"DBEEL_EXTRACT_PERSIST": "0"},
    "persist1": {"DBEEL_EXTRACT_PERSIST": "1"},
    "pdl": {"DBEEL_PDL": "1"},
    "pdl-fused0-persist1": {"DBEEL_PDL": "1", "DBEEL_FUSED_FINAL": "0", "DBEEL_EXTRACT_PERSIST": "1"},
    "events0": {"DBEEL_STAGE_EVENTS": "0"},
    "taper0": {"DBEEL_PARTITION_TAPER": "0"},  # only the host pipeline cuts partitions
}
# host pipeline and compact_stream: even small jobs become many key-range partitions
TINY_PARTITIONS = {"DBEEL_PIPELINE_MIN_KB": "1", "DBEEL_PARTITION_KB": "24"}
KERNEL_SPECS = ["narrow0", "narrow0-fused0", "fused0", "persist0", "persist1", "pdl", "pdl-fused0-persist1"]
COMPACTION_SPECS = KERNEL_SPECS + ["events0"]
EXTRACT_PERSIST_DEFAULT = 6  # dbeel_engine::extract_persist
EXTRACT_STEP = 512           # entries per CTA and step of k_extract: 256 threads x kExtractEPT


def _env(spec, **extra):
    """The variables of an engine: the original fixture's, then the spec's (which win)."""
    return {**extra, **SPECS[spec]}


# ---- engines: every fixture is class-scoped and keyed by the class's spec, so a class builds and closes one spec's engines
# at a time

@pytest.fixture(scope="class")
def spec(request):
    return request.param


@pytest.fixture(scope="class")
def spec_engine(spec):
    eng = _engine(_env(spec))
    yield eng
    eng.close()


@pytest.fixture(scope="class")
def spec_partition_engine(spec):
    """test_gpu_parity's tiny_partition_engine under the spec."""
    eng = _engine(_env(spec, **TINY_PARTITIONS))
    yield eng
    eng.close()


@pytest.fixture(scope="class")
def spec_one_cta_engine(spec):
    """test_gpu_merge_final_pipeline's engine_one_cta under the spec."""
    eng = _engine(_env(spec, DBEEL_FUSED_FINAL="1", DBEEL_FIN_CTAS_RT="1"))
    yield eng
    eng.close()


@pytest.fixture
def spec_monkeypatch(spec, monkeypatch):
    """For tests that build their own engines: the spec's variables are set while they run."""
    for k, v in SPECS[spec].items():
        monkeypatch.setenv(k, v)
    return monkeypatch


@pytest.fixture
def spec_leaf_engine(spec, monkeypatch):
    """test_gpu_reader's / test_gpu_get_values_stream's tiny_engine (4 KB leaf groups) under the spec."""
    monkeypatch.delenv("DBEEL_PARTITION_MB", raising=False)
    eng = _engine(_env(spec, DBEEL_PARTITION_KB="4"))
    yield eng
    eng.close()


@pytest.fixture
def spec_make_engine(spec, monkeypatch):
    """test_gpu_scan_stream's make_engine under the spec."""
    monkeypatch.delenv("DBEEL_PARTITION_MB", raising=False)
    made = []

    def make(budget_kb: int, ring: int = 3):
        made.append(_engine(_env(spec, DBEEL_PARTITION_KB=str(budget_kb), DBEEL_STREAM_RING=str(ring))))
        return made[-1]

    yield make
    for e in made:
        e.close()


@pytest.fixture(scope="module")
def dev():
    import torch
    return torch.device("cuda:0")


# the fixtures of the existing tests -> the spec's engines that replace them
FIXTURES = {
    "engine": "spec_engine",
    "fused_engine": "spec_engine",           # FUSED_FINAL=1 is the engine default
    "engine_default_ctas": "spec_engine",
    "engine_one_cta": "spec_one_cta_engine",
    "tiny_partition_engine": "spec_partition_engine",
    "tiny_engine": "spec_leaf_engine",
    "make_engine": "spec_make_engine",
    "monkeypatch": "spec_monkeypatch",
}


def rerun(fn, **subset):
    """A test method that calls the existing test `fn` with the spec's engines in place of its engine fixtures (FIXTURES)
    and keeps its parametrizations; `subset` narrows a parametrization (by its argnames) to the values given."""
    names = list(inspect.signature(fn).parameters)
    ours = [FIXTURES.get(n, n) for n in names]

    def test(self, **kw):
        fn(**{n: kw[o] for n, o in zip(names, ours)})

    P = inspect.Parameter
    test.__signature__ = inspect.Signature([P("self", P.POSITIONAL_OR_KEYWORD)] +
                                           [P(o, P.KEYWORD_ONLY) for o in dict.fromkeys(ours)])
    test.__name__ = test.__qualname__ = fn.__name__
    test.__doc__ = fn.__doc__
    marks = []
    for m in getattr(fn, "pytestmark", []):
        if m.name == "parametrize":
            marks.append(pytest.mark.parametrize(m.args[0], subset.pop(m.args[0], m.args[1]), **m.kwargs).mark)
    assert not subset, f"{fn.__name__} has no parametrization {list(subset)}"
    test.pytestmark = marks
    return test


def on_specs(names):
    return pytest.mark.parametrize("spec", names, indirect=True)


# ---- 1. each spec runs the kernels it claims

def _k(name, *targs, prefix=False):
    """Regex for a kernel in a demangled name, whitespace-tolerant: _k("k_extract", "true", "false") matches
    `void dbeel::k_extract<true, false>(dbeel::Params, int)`; prefix=True leaves the argument list open."""
    if not targs:
        return re.compile(r"\b" + name + r"\b")
    body = r"\s*,\s*".join(targs)
    return re.compile(r"\b" + name + r"<\s*" + body + (r"\s*[,>]" if prefix else r"\s*>"))


def _expected_kernels(env, flush):
    """(kernels that must run, kernels that must not) for one job on an engine with these variables."""
    narrow = env.get("DBEEL_NARROW", "1") != "0"
    fused = env.get("DBEEL_FUSED_FINAL", "1") != "0" and not flush  # only single compactions take k_merge_final
    persist = int(env.get("DBEEL_EXTRACT_PERSIST", str(EXTRACT_PERSIST_DEFAULT))) > 0
    n, other = ("true", "false") if narrow else ("false", "true")
    want = [_k("k_copy_words"), _k("k_gather_h"), _k("k_extract", n, "false", "true" if narrow and persist else "false")]
    banned = [_k("k_extract", other, prefix=True), _k("k_merge_final", other), _k("k_resolve", other)]
    if narrow and not persist:
        banned.append(_k("k_extract", "true", "false", "true"))
    tail = [_k("k_resolve", n), _k("k_scan_tiles"), _k("k_scan_chunks"), _k("k_emit")]
    if fused:
        want.append(_k("k_merge_final", n))
        banned += tail
    else:
        want += tail
        banned.append(_k("k_merge_final"))
    return want, banned


def _kernel_names(job):
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        job()
        torch.cuda.synchronize()
    return {ev.key for ev in prof.key_averages()}


@pytest.mark.gpu
@on_specs([s for s in SPECS if s != "taper0"])
class TestKernelIdentity:
    def test_each_spec_runs_the_kernels_it_names(self, spec, spec_engine):
        """One clean 2-run compaction and one flush under torch.profiler; the demangled kernel names must show the
        instantiations the spec selects and none of the ones it replaces.  DBEEL_PDL (a launch attribute) and
        DBEEL_STAGE_EVENTS (event records between the kernels) change no kernel name: for those the check is that the
        kernels are the default's, and for STAGE_EVENTS=0 that the stage times read 0."""
        env = SPECS[spec]
        runs = [sstable.build_run([(b"k%06d" % n, b"v%d" % r * (n % 9), BASE_TS + r) for n in range(r, 6000, 1 + r)])
                for r in range(2)]
        arrivals = sstable.build_run([(b"k%04d" % (n * 7 % 1000), b"x" * (n % 13), BASE_TS - n) for n in range(5000)])
        jobs = {"compaction": lambda: check_against_oracle(spec_engine, runs, False, what=spec),
                "flush": lambda: spec_engine.flush(arrivals)}
        for what, job in jobs.items():
            names = _kernel_names(job)
            assert any(_k("k_copy_words").search(n) for n in names), f"{what}: the profiler recorded no kernel of the job"
            want, banned = _expected_kernels(env, flush=what == "flush")
            for pat in want:
                assert any(pat.search(n) for n in names), f"{spec} {what}: no kernel matches {pat.pattern} in {sorted(names)}"
            for pat in banned:
                hit = [n for n in names if pat.search(n)]
                assert not hit, f"{spec} {what}: {hit} ran"
        spec_engine.compact(runs, False, seed=SEED)
        st = spec_engine.stats()
        stage_ms = [st["ms_extract"], st["ms_merge"], st["ms_resolve"], st["ms_gather"]]
        if env.get("DBEEL_STAGE_EVENTS") == "0":
            assert stage_ms == [0, 0, 0, 0]
        else:
            assert st["ms_extract"] > 0 and st["ms_gather"] > 0, stage_ms
        assert st["ms_total"] > 0


# ---- 2. the parity corpus under every spec that changes a compaction kernel or its launch

@pytest.mark.gpu
@on_specs(COMPACTION_SPECS)
class TestCompactionFamily:
    test_cfg1_two_way_1k_keys = rerun(parity.test_cfg1_two_way_1k_keys)
    test_get_after_compaction = rerun(parity.test_get_after_compaction)
    test_adversarial_keys_match_oracle_and_model = rerun(parity.test_adversarial_keys_match_oracle_and_model, seed=[0, 3, 5])
    test_tie_breaks = rerun(parity.test_tie_breaks)
    test_tombstones = rerun(parity.test_tombstones)
    test_empty_and_ragged_inputs = rerun(parity.test_empty_and_ragged_inputs)
    test_truncated_and_corrupt_runs_end_silently = rerun(parity.test_truncated_and_corrupt_runs_end_silently)
    test_index_fields_are_verified_not_ignored = rerun(parity.test_index_fields_are_verified_not_ignored)
    test_long_shared_prefixes_and_window_ties = rerun(parity.test_long_shared_prefixes_and_window_ties)
    test_common_prefix_longer_than_the_cap = rerun(parity.test_common_prefix_longer_than_the_cap)
    test_bloom_small = rerun(parity.test_bloom_small)
    test_variable_key_lengths_in_bloom = rerun(parity.test_variable_key_lengths_in_bloom)
    test_unsorted_run_is_refused = rerun(parity.test_unsorted_run_is_refused)
    test_large_and_tiny_entries_mixed = rerun(parity.test_large_and_tiny_entries_mixed)
    test_three_hundred_small_runs = rerun(parity.test_three_hundred_small_runs)
    test_multi_megabyte_entries_and_keys = rerun(parity.test_multi_megabyte_entries_and_keys)
    test_flush_matches_memtable = rerun(parity.test_flush_matches_memtable)
    test_flush_large_zipf_batch = rerun(parity.test_flush_large_zipf_batch)
    test_flush_many_equals_separate_flushes = rerun(parity.test_flush_many_equals_separate_flushes)
    test_compact_many_equals_separate_compactions = rerun(parity.test_compact_many_equals_separate_compactions, seed=[1, 2])
    test_compact_many_edge_shapes = rerun(parity.test_compact_many_edge_shapes)
    test_device_resident_entry_point = rerun(parity.test_device_resident_entry_point)
    test_flush_device_entry_point = rerun(parity.test_flush_device_entry_point)
    test_async_submit_poll_wait = rerun(parity.test_async_submit_poll_wait)

    # test_fused_adversarial_keys is left out: it asserts the fused path's launch count, which FUSED_FINAL=0 changes
    test_fused_edge_shapes = rerun(merge_final.test_fused_edge_shapes)
    test_groups_straddling_merge_tiles = rerun(merge_final.test_groups_straddling_merge_tiles, seed=[0, 2])
    test_fused_reference_reader_and_host_pipeline = rerun(merge_final.test_fused_reference_reader_and_host_pipeline)
    test_one_and_two_tiles = rerun(merge_final_pipeline.test_one_and_two_tiles)

    test_wrong_key_size_is_ignored = rerun(reference_reader.test_wrong_key_size_is_ignored)
    test_wrong_offsets_are_ignored = rerun(reference_reader.test_wrong_offsets_are_ignored)
    test_full_size_is_what_positions_the_stream = rerun(reference_reader.test_full_size_is_what_positions_the_stream)
    test_timestamp_range_ends_the_run = rerun(reference_reader.test_timestamp_range_ends_the_run)
    test_timestamp_of_unique_and_duplicate_keys = rerun(reference_reader.test_timestamp_of_unique_and_duplicate_keys)
    test_clean_inputs_take_the_fast_path_and_match_the_default_mode = rerun(
        reference_reader.test_clean_inputs_take_the_fast_path_and_match_the_default_mode)
    test_random_index_damage_matches_the_oracle = rerun(reference_reader.test_random_index_damage_matches_the_oracle)

    # exact caps: every residue mod 16 is in the first 16 cases; the tile edges and the megabyte jobs follow
    test_compact_device_fills_exact_caps = rerun(edges.test_compact_device_fills_exact_caps,
                                                 case=[0, 3, 6, 9, 13, 15] + list(range(16, len(edges.COMPACT_CASES))))
    test_inputs_placed_at_any_byte_with_poison_around = rerun(edges.test_inputs_placed_at_any_byte_with_poison_around,
                                                              shift=[0, 1, 7, 8, 15, 33, 4097])

    test_replay_of_a_write_heavy_log = rerun(wal.test_replay_of_a_write_heavy_log)
    test_adversarial_keys_sizes_and_padding = rerun(wal.test_adversarial_keys_sizes_and_padding, seed=[0, 1])
    test_records_that_hide_records = rerun(wal.test_records_that_hide_records)
    test_zero_pages_torn_tails_corrupt_lengths_bad_timestamps = rerun(wal.test_zero_pages_torn_tails_corrupt_lengths_bad_timestamps)
    test_capacity_is_enforced_like_the_tree = rerun(wal.test_capacity_is_enforced_like_the_tree)
    test_device_resident_log = rerun(wal.test_device_resident_log)


@pytest.mark.gpu
@on_specs(COMPACTION_SPECS + ["taper0"])
class TestHostPipeline:
    """The host entry point's key-range partitions and dbeel_compact_stream: every partition is a compaction job."""
    test_pipelined_host_path_is_byte_identical = rerun(parity.test_pipelined_host_path_is_byte_identical, seed=[0, 1])
    test_pipelined_path_falls_back_on_corrupt_input = rerun(parity.test_pipelined_path_falls_back_on_corrupt_input)
    test_compact_stream_equals_compact_and_the_oracle = rerun(parity.test_compact_stream_equals_compact_and_the_oracle,
                                                              seed=[0, 1])
    test_pipelined_host_path_falls_back = rerun(reference_reader.test_pipelined_host_path_falls_back)


@pytest.mark.gpu
@on_specs(KERNEL_SPECS)
class TestScaledShapes:
    test_scaled_benchmark_shapes = rerun(parity.test_scaled_benchmark_shapes)


@pytest.mark.gpu
@on_specs(["pdl"])
class TestEveryLaunchUnderPdl:
    """Scans, reads, readers, routing and the cfg5 pipeline launch through the same launch_k: with DBEEL_PDL=1 only
    griddepcontrol.wait orders each kernel after its predecessor."""
    test_hash_ranges_match_oracle = rerun(scan.test_hash_ranges_match_oracle)
    test_key_ranges_match_oracle = rerun(scan.test_key_ranges_match_oracle)
    test_damaged_trees_stop_where_the_reference_stops = rerun(scan.test_damaged_trees_stop_where_the_reference_stops)
    test_host_and_device_entry_points_agree = rerun(scan.test_host_and_device_entry_points_agree)
    test_output_feeds_dbeel_flush = rerun(scan.test_output_feeds_dbeel_flush)
    test_capacity_and_arguments = rerun(scan.test_capacity_and_arguments)
    test_compaction_after_scans_is_unchanged = rerun(scan.test_compaction_after_scans_is_unchanged)
    test_tree_scan_on_files = rerun(scan.test_tree_scan_on_files)
    test_output_larger_than_the_inputs = rerun(scan.test_output_larger_than_the_inputs)
    test_error_paths = rerun(scan.test_error_paths)

    test_hash_ranges_match_oracle_and_dbeel_scan = rerun(scan_stream.test_hash_ranges_match_oracle_and_dbeel_scan, ring=[2])
    test_stream_key_ranges_match_oracle = rerun(scan_stream.test_key_ranges_match_oracle)
    test_budgets_from_one_record_to_more_than_the_tree = rerun(scan_stream.test_budgets_from_one_record_to_more_than_the_tree)
    test_entry_larger_than_the_budget_and_overlapping_records = rerun(
        scan_stream.test_entry_larger_than_the_budget_and_overlapping_records)
    test_damage_in_every_partition_position = rerun(scan_stream.test_damage_in_every_partition_position)
    test_callback_errors_come_back_and_the_engine_stays_usable = rerun(
        scan_stream.test_callback_errors_come_back_and_the_engine_stays_usable)
    test_tree_scan_stream_on_files = rerun(scan_stream.test_tree_scan_stream_on_files)
    test_compaction_after_streamed_scans_is_unchanged = rerun(scan_stream.test_compaction_after_streamed_scans_is_unchanged)

    test_both_modes_on_a_compacted_table_with_a_filter = rerun(get_values.test_both_modes_on_a_compacted_table_with_a_filter)
    test_get_values_tiny_tables = rerun(get_values.test_tiny_tables_and_the_reference_early_exit)
    test_four_overlapping_tables_newest_first = rerun(get_values.test_four_overlapping_tables_newest_first)
    test_tombstones_empty_values_and_entries_larger_than_a_gather_tile = rerun(
        get_values.test_tombstones_empty_values_and_entries_larger_than_a_gather_tile)
    test_nothing_found_no_keys_no_tables = rerun(get_values.test_nothing_found_no_keys_no_tables)
    test_bad_entries_and_corrupt_records = rerun(get_values.test_bad_entries_and_corrupt_records)
    test_device_entry_point_on_compact_device_output_with_guards_and_caps = rerun(
        get_values.test_device_entry_point_on_compact_device_output_with_guards_and_caps)
    test_device_inputs_from_flush_many_device_unaligned_data = rerun(
        get_values.test_device_inputs_from_flush_many_device_unaligned_data)
    test_output_is_an_arrival_batch_dbeel_flush_takes = rerun(get_values.test_output_is_an_arrival_batch_dbeel_flush_takes)
    test_tree_get_values_after_flush_and_compact = rerun(get_values.test_tree_get_values_after_flush_and_compact)

    test_parity_with_get_values_on_every_table_set = rerun(get_values_stream.test_parity_with_get_values_on_every_table_set)
    test_stream_damage_at_fences_and_inside_leaves = rerun(get_values_stream.test_damage_at_fences_and_inside_leaves)
    test_a_table_the_filter_rejects_is_not_read = rerun(get_values_stream.test_a_table_the_filter_rejects_is_not_read)
    test_sparse_batch_reads_a_small_share_and_a_dense_one_reads_data_once = rerun(
        get_values_stream.test_sparse_batch_reads_a_small_share_and_a_dense_one_reads_data_once)
    test_callback_errors_and_capacity = rerun(get_values_stream.test_callback_errors_and_capacity)
    test_a_table_larger_than_device_memory = rerun(get_values_stream.test_a_table_larger_than_device_memory)
    test_tree_get_values_stream_after_flush_and_compact = rerun(
        get_values_stream.test_tree_get_values_stream_after_flush_and_compact)

    test_parity_on_every_case = rerun(reader.test_parity_on_every_case)
    test_reader_damage_at_fences_and_inside_leaves = rerun(reader.test_damage_at_fences_and_inside_leaves)
    test_reads_from_the_second_batch_on = rerun(reader.test_reads_from_the_second_batch_on)
    test_fallbacks_read_fences_per_call = rerun(reader.test_fallbacks_read_fences_per_call)
    test_callback_errors_and_capacity_leave_the_reader_usable = rerun(
        reader.test_callback_errors_and_capacity_leave_the_reader_usable)
    test_tree_reader_snapshots = rerun(reader.test_tree_reader_snapshots)
    test_device_memory_is_the_filters_and_the_fence_budget = rerun(reader.test_device_memory_is_the_filters_and_the_fence_budget)

    test_reference_loop_on_a_compacted_table_with_bloom = rerun(lookup.test_reference_loop_on_a_compacted_table_with_bloom)
    test_exact_mode_finds_every_present_key = rerun(lookup.test_exact_mode_finds_every_present_key)
    test_newest_table_answers_first_and_filters_are_counted = rerun(
        lookup.test_newest_table_answers_first_and_filters_are_counted)
    test_device_resident_lookup_on_compaction_output = rerun(lookup.test_device_resident_lookup_on_compaction_output)
    test_malformed_inputs_are_reported = rerun(lookup.test_malformed_inputs_are_reported)

    test_route_device_matches_the_oracle = rerun(routing.test_route_device_matches_the_oracle)
    test_route_then_sparse_flush_equals_flushing_each_shards_stream = rerun(
        routing.test_route_then_sparse_flush_equals_flushing_each_shards_stream)
    test_device_memtable_cuts_match_the_host_trigger = rerun(routing.test_device_memtable_cuts_match_the_host_trigger)
    # the two single-rank shapes: the other two add ranks and size, not launches
    test_cfg5_pipeline_matches_the_oracle = rerun(cfg5_tests.test_cfg5_pipeline_matches_the_oracle,
                                                  **{"n_writes,capacity,factor,wave,world": [(90_000, 300, 2, 3, 1),
                                                                                             (40_000, 8192, 8, 8, 1)]})


# ---- 3. the persistent extract's step and wave borders
#
# k_extract<.., kPersist> runs one resident wave of sm_count x EXTRACT_PERSIST CTAs; each thread walks steps of W entries
# and fetches the next step's index records (and their predecessors, for the running-offset check) a step ahead.  These
# jobs put a run border, an empty run, wrong offsets and cross-border duplicates at the step borders of that walk.

def _wave(persist):
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count * persist * EXTRACT_STEP


def _border_run(seed, n, id_space, equal_ts):
    """n sorted distinct 17-byte keys out of id_space ids (so runs share keys), 8-byte docs, 2 % tombstones."""
    rng = np.random.default_rng(seed)
    ids = np.sort(rng.choice(max(id_space, n), n, replace=False))
    ts = np.full(n, BASE_TS, np.int64) if equal_ts else BASE_TS + rng.integers(0, 3, n)
    return sstable.build_run_fixed(W.format_keys(ids), rng.integers(0, 256, (n, 8), dtype=np.uint8), ts, rng.random(n) < 0.02)


def _with_bad_offset(run, i):
    """Record i's offset off by one: the engine ends the run there.  Returns the damaged run and the valid prefix."""
    d, ix = run
    bad = ix.copy()
    bad[16 * i] ^= 1
    return (d, bad), (d, ix[:16 * i])


def _border_case(w, n, layout):
    """(runs the engine gets, runs with the damage cut off -- what it must compact, number of runs it must cut short) for
    a job of n index records whose extract walks steps of w entries."""
    # cuts: (first global position, last + 1, local index of a wrong offset or None, id space, equal timestamps)
    if layout == "run_at_border":
        # ... | run ending at w | empty run | run starting at w | ...; the runs on either side share keys at equal timestamps
        a = max(0, w - 700)
        cuts = [(0, min(n, a), None, 5 * a // 4, False), (a, min(n, w), None, 2000, True), (w, w, None, 0, True),
                (w, max(n, w), None, 2000, True)]
    else:
        # a wrong offset at position w (fetched a step ahead, the first record of step 1) and another in step 2
        a, b = w - 1000, w + 2000
        third = 2 * w + 300 if n > 2 * w + 300 else 2 * w
        cuts = [(0, a, None, 5 * a // 4, False), (a, min(n, b), w - a, 4000, True)]
        if n > b:
            cuts.append((b, n, third - b if n > third else None, 5 * (n - b) // 4, True))
    runs, clean, cut_short = [], [], 0
    for k, (lo, hi, bad, space, eq) in enumerate(cuts):
        run = _border_run([w, n, k, len(layout)], hi - lo, space, eq)
        if bad is not None and bad < hi - lo:
            damaged, prefix = _with_bad_offset(run, bad)
            runs.append(damaged)
            clean.append(prefix)
            cut_short += 1
        else:
            runs.append(run)
            clean.append(run)
    assert sum(i.size // 16 for _, i in runs) == n
    return runs, clean, cut_short


_BORDER_EXPECTED = {}


def _digest(a):
    return None if a is None else hashlib.blake2b(np.ascontiguousarray(a).data).hexdigest()


def _border_expected(key, clean, keep, bloom_min_size):
    """Digests of the oracle's output for the clean runs (checked once against the Python model), cached across specs:
    the oracle and the model are the slow side."""
    if key not in _BORDER_EXPECTED:
        od, oi, ob, on = oracle.compact(clean, keep, bloom_min_size=bloom_min_size, seed=SEED)
        exp, mn = model_compact(clean, keep)
        assert on == mn
        assert_run_equal((od, oi), exp, f"{key}: oracle vs model")
        _BORDER_EXPECTED[key] = (on, _digest(od), _digest(oi), _digest(ob))
    return _BORDER_EXPECTED[key]


def _persist_of(spec):
    p = int(SPECS[spec].get("DBEEL_EXTRACT_PERSIST", str(EXTRACT_PERSIST_DEFAULT)))
    return p if p > 0 else EXTRACT_PERSIST_DEFAULT  # no persistent wave: the default's borders, as plain positions


# total index records of a job, from the wave W
BORDER_TOTALS = {"W-1": lambda w: w - 1, "W": lambda w: w, "W+1": lambda w: w + 1, "W+511": lambda w: w + 511,
                 "W+512": lambda w: w + 512, "W+513": lambda w: w + 513, "2W+1": lambda w: 2 * w + 1,
                 "2W+700": lambda w: 2 * w + 700}
BORDER_CASES = ([("run_at_border", at) for at in BORDER_TOTALS] +
                [("bad_offsets", at) for at in BORDER_TOTALS if at not in ("W-1", "W")])  # the bad record sits at W


@pytest.mark.gpu
@on_specs(["default", "persist1", "persist0", "narrow0"])
class TestExtractWaveBorders:
    @pytest.mark.parametrize("layout,at", BORDER_CASES)
    def test_compaction_across_the_wave(self, spec, spec_engine, layout, at):
        w = _wave(_persist_of(spec))
        n = BORDER_TOTALS[at](w)
        runs, clean, cut_short = _border_case(w, n, layout)
        keep = layout == "bad_offsets"
        # a filter is sized by the input's record count, so only the undamaged layout (same records either way) has one
        bms = capi.DEFAULT_BLOOM_MIN_SIZE if cut_short == 0 else 1 << 40
        on, dd, di, db = _border_expected((w, n, layout), clean, keep, bms)
        gd, gi, gb, gn = spec_engine.compact(runs, keep_tombstones=keep, bloom_min_size=bms, seed=SEED)
        st = spec_engine.stats()
        # one job, not key-range partitions: the extract sees all n records
        assert st["partitions"] == 1 and st["entries_in"] == n and st["runs_truncated"] == cut_short
        assert gn == on, f"{layout} N={at} (W={w}): items {gn} != {on}"
        if (_digest(gd), _digest(gi)) != (dd, di):
            od, oi, _, _ = oracle.compact(clean, keep, bloom_min_size=bms, seed=SEED)
            assert_run_equal((gd, gi), (od, oi), f"{layout} N={at} (W={w})")
        assert _digest(gb) == db, f"{layout} N={at} (W={w}): .bloom differs"

    def test_flush_of_w_plus_one_arrivals(self, spec, spec_engine):
        w = _wave(_persist_of(spec))
        rng = np.random.default_rng(w)
        ids = rng.integers(0, w // 3, w + 1)
        ts = BASE_TS + np.where(rng.random(w + 1) < 0.5, 0, rng.integers(-5, 5, w + 1))  # repeats at equal timestamps
        batch = sstable.build_run_fixed(W.format_keys(ids), rng.integers(0, 256, (w + 1, 8), dtype=np.uint8), ts,
                                        rng.random(w + 1) < 0.02)
        key = (w, "flush")
        if key not in _BORDER_EXPECTED:
            (od, oi, on), = oracle.memtable_flushes(batch, capacity=1 << 20)
            assert_run_equal((od, oi), model_flush(batch, 1 << 20)[0], "oracle vs model")
            _BORDER_EXPECTED[key] = (on, _digest(od), _digest(oi))
        on, dd, di = _BORDER_EXPECTED[key]
        gd, gi, gn = spec_engine.flush(batch)
        assert gn == on
        if (_digest(gd), _digest(gi)) != (dd, di):
            (od, oi, _), = oracle.memtable_flushes(batch, capacity=1 << 20)
            assert_run_equal((gd, gi), (od, oi), f"flush of {w + 1} arrivals")


# ---- 4. the settings no other file sets

@pytest.mark.gpu
def test_pipeline_off_compacts_above_the_threshold_in_one_piece():
    """DBEEL_PIPELINE=0: a host compaction above pipeline_min_bytes runs as one job (the same job cuts into partitions with
    the pipeline on)."""
    rng = np.random.default_rng(12)
    pool = [b"\xb0k%015d" % n for n in range(20_000)]
    runs = random_runs(rng, 5, [3000, 2500, 4000, 100, 3500], pool, max_doc=150)
    for env, parts in (({"DBEEL_PIPELINE": "0"}, lambda p: p == 1), ({}, lambda p: p > 4)):
        eng = _engine({**TINY_PARTITIONS, **env})
        try:
            for keep in (False, True):
                gd, gi, _, n = check_against_oracle(eng, runs, keep, bloom_min_size=10_000, what=f"{env} keep={keep}")
                assert parts(eng.stats()["partitions"]), (env, eng.stats()["partitions"])
                exp, en = model_compact(runs, keep)
                assert n == en
                assert_run_equal((gd, gi), exp, f"{env} vs model")
        finally:
            eng.close()


@pytest.mark.gpu
def test_partition_size_in_megabytes():
    """DBEEL_PARTITION_MB: 1 MB partitions of a 4.6 MB host compaction."""
    eng = _engine({"DBEEL_PIPELINE_MIN_KB": "1", "DBEEL_PARTITION_MB": "1"})
    try:
        c = W.scaled(W.CFG2, 2000)
        check_against_oracle(eng, W.make_merge_runs(c), False, what="1 MB partitions")
        assert eng.stats()["partitions"] > 2
    finally:
        eng.close()


@pytest.mark.gpu
def test_streamed_tree_compaction_writes_through_pwrite(monkeypatch, tmp_path):
    """DBEEL_STREAM_MMAP=0 (read per call): the streamed tree compaction writes its output files with pwrite instead of
    through a mapping; same files as the oracle's."""
    monkeypatch.setenv("DBEEL_STREAM_MMAP", "0")
    host_tree.test_streamed_compaction_is_byte_identical(monkeypatch, tmp_path, 2)


# ---- 5. no setting without a test (CPU)

# variables read by the native code that a test elsewhere sets
TESTED_ELSEWHERE = {
    "FIN_CTAS_RT": "test_gpu_merge_final_pipeline",
    "PARTITION_KB": "test_gpu_parity",
    "PIPELINE_MIN_KB": "test_gpu_parity",
    "IO_THREADS": "test_host_tree",
    "TREE_STREAM": "test_host_tree",
    "STREAM_RING": "test_gpu_scan_stream",
    "PIPELINE": "test_gpu_engine_settings",       # test_pipeline_off_compacts_above_the_threshold_in_one_piece
    "PARTITION_MB": "test_gpu_engine_settings",   # test_partition_size_in_megabytes
    "STREAM_MMAP": "test_gpu_engine_settings",    # test_streamed_tree_compaction_writes_through_pwrite
}
PRINT_ONLY = {"TRACE"}  # a per-partition timeline on stderr; changes nothing the engine computes


def native_settings(root=os.path.join(ROOT, "dbeel_b200", "csrc")):
    """Every DBEEL_* name the native sources pass to getenv."""
    found = set()
    for d, _, files in os.walk(root):
        for f in files:
            if f.endswith((".cu", ".cuh", ".cc", ".h", ".cpp", ".hpp")):
                with open(os.path.join(d, f), encoding="utf-8") as fh:
                    found.update(re.findall(r'getenv\(\s*"DBEEL_(\w+)"\s*\)', fh.read()))
    return found


def test_every_native_setting_has_a_test():
    matrix = {k[len("DBEEL_"):] for env in list(SPECS.values()) + [TINY_PARTITIONS] for k in env}
    read = native_settings()
    assert read, "no getenv(\"DBEEL_...\") found: the scan is broken"
    untested = sorted(read - matrix - set(TESTED_ELSEWHERE) - PRINT_ONLY)
    assert not untested, (f"{', '.join('DBEEL_' + n for n in untested)}: read by the engine but set by no test; add a spec "
                          "to SPECS, or a test and its entry in TESTED_ELSEWHERE")
    stale = sorted((matrix | set(TESTED_ELSEWHERE) | PRINT_ONLY) - read)
    assert not stale, f"{', '.join('DBEEL_' + n for n in stale)}: listed here but no longer read by the engine"
    for name, module in TESTED_ELSEWHERE.items():
        with open(os.path.join(ROOT, "tests", module + ".py"), encoding="utf-8") as fh:
            assert f'"DBEEL_{name}"' in fh.read(), f"{module} does not set DBEEL_{name}"
