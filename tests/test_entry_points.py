"""CPU-side check of what each entry point of the public headers (include/chd_gpu*.h) does before it touches the engine: the lock,
the device, the copy wait and the fetch guard (the rules: ENTRY_* in channeld_b200/csrc/chd_engine.h), and whether it is refused
while a chd_begin_interest is pending (rule 13 of DESIGN.md §5).  Every entry point declares its needs once, with CHD_ENTER, and
NEEDS below is the inventory of those declarations; CHAIN is the inventory of rule 13's callers.  A change to either shows up here.
Reads the sources only: runs without a GPU and without a build.

An entry point here is a function of a header that takes a `chd_engine*` and returns a chd_status.  Left out: the functions
that take a `const chd_engine*`, which read host fields only, and chd_destroy, which releases the engine whatever fails."""
import glob
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "channeld_b200", "csrc")
HEADERS = ["chd_gpu.h", "chd_gpu_subs.h", "chd_gpu_facing.h", "chd_gpu_rings.h"]

NEEDS = {
    # chd_engine.cu
    "chd_set_stream": "DEVICE",
    "chd_sync": "COPY_WAIT",
    "chd_enable_graphs": "0",
    "chd_profile_enable": "COPY_WAIT",
    "chd_profile_timeline": "COPY_WAIT",
    "chd_profile_get": "COPY_WAIT",
    # chd_entities.cu
    "chd_cell_of_valid": "LOCK|DEVICE",
    "chd_set_entities": "DEVICE",
    "chd_prefetch_entities": "DEVICE",
    "chd_set_entities_f32": "DEVICE",
    "chd_prefetch_entities_f32": "DEVICE",
    "chd_entity_buffers": "0",
    "chd_set_entity_count": "0",
    "chd_set_entity_ids": "DEVICE",
    "chd_assign_cells": "FETCH_GUARD",
    "chd_build": "COPY_WAIT|FETCH_GUARD",
    # chd_interest.cu
    "chd_prefetch_queries": "LOCK|DEVICE",
    "chd_set_subscribers": "COPY_WAIT",
    "chd_add_subscribers": "LOCK|DEVICE",
    "chd_remove_subscribers": "LOCK|DEVICE",
    "chd_query_channel_ids": "LOCK|DEVICE",
    "chd_update_interest": "COPY_WAIT|FETCH_GUARD",
    # chd_tick.cu
    "chd_emit_visible": "COPY_WAIT|FETCH_GUARD",
    "chd_set_channel_start_times": "DEVICE",
    "chd_fanout_tick": "COPY_WAIT|FETCH_GUARD",
    "chd_adopt_prefetched": "DEVICE",
    "chd_summary": "COPY_WAIT",
    "chd_begin_interest": "FETCH_GUARD",
    "chd_tick": "FETCH_GUARD",
    # chd_rings.cu
    "chd_set_rings": "DEVICE",
    "chd_prefetch_rings": "DEVICE",
    "chd_rings_init": "DEVICE",
    "chd_rings_append": "DEVICE",
    "chd_get_rings": "COPY_WAIT",
    # chd_results.cu
    "chd_get_cells": "COPY_WAIT",
    "chd_get_pairs": "COPY_WAIT",
    "chd_get_query_status": "COPY_WAIT",
    "chd_get_diff": "COPY_WAIT",
    "chd_get_visible": "COPY_WAIT",
    "chd_get_visible_slot": "COPY_WAIT",
    "chd_get_due": "COPY_WAIT",
    "chd_get_handover": "COPY_WAIT",
    "chd_fetch_results_delta": "DEVICE",
    "chd_fetch_results_async_delta": "DEVICE",
    "chd_fetch_wait_delta": "DEVICE",
    "chd_device_view": "COPY_WAIT",
    # chd_delta.cu
    "chd_reserve_visible_delta": "DEVICE",
    "chd_reserve_visible_delta_ids": "DEVICE",
    "chd_visible_delta": "FETCH_GUARD",
    "chd_get_visible_delta": "COPY_WAIT",
    # chd_table.cu
    "chd_entity_table_init": "DEVICE",
    "chd_spawn_entities": "DEVICE",
    "chd_spawn_entities_f32": "DEVICE",
    "chd_despawn_entities": "DEVICE",
    "chd_move_entities": "DEVICE",
    "chd_move_entities_f32": "DEVICE",
    "chd_get_entity_stats": "COPY_WAIT",
    "chd_handoff_entities": "DEVICE",
    # chd_follow.cu
    "chd_follow_bind": "LOCK|DEVICE",
    "chd_follow_unbind": "LOCK|DEVICE",
    "chd_follow_queries": "LOCK|DEVICE",
    "chd_follow_queries_with": "LOCK|DEVICE",
    "chd_get_follow": "LOCK|COPY_WAIT",
    # chd_shard.cu
    "chd_set_slab": "0",
    "chd_export_border": "FETCH_GUARD",
    "chd_import_halo": "DEVICE",
    "chd_comm_init": "DEVICE",
    "chd_comm_destroy": "DEVICE",
    "chd_tick_sharded": "COPY_WAIT|FETCH_GUARD",
    "chd_comm_use_collective": "0",
    "chd_migrate_out": "LOCK|DEVICE",
    "chd_migrate_in": "LOCK|DEVICE",
    "chd_get_rehome": "COPY_WAIT",
    # chd_extras.cu
    "chd_due_classes": "COPY_WAIT",
    "chd_set_subscriber_types": "LOCK|DEVICE",
    "chd_adjacent_broadcast": "LOCK|COPY_WAIT",
    # chd_payload.cu
    "chd_set_payload_bytes": "LOCK|COPY_WAIT",
    "chd_assemble_payloads": "LOCK|COPY_WAIT",
    "chd_frame_packets": "LOCK|COPY_WAIT",
    # chd_gpu_subs.h: chd_apply_subscriptions takes the lock besides chd_update_interest's needs: it opens epochs of the query
    # stage's scan sites, which chd_query_channel_ids bumps from any thread
    "chd_apply_subscriptions": "LOCK|COPY_WAIT|FETCH_GUARD",
    # chd_gpu_facing.h: the event calls as their chd_gpu.h counterparts, set-frame as chd_follow_bind, get-frame as chd_get_follow
    "chd_spawn_entities_facing": "DEVICE",
    "chd_spawn_entities_facing_f32": "DEVICE",
    "chd_move_entities_facing": "DEVICE",
    "chd_move_entities_facing_f32": "DEVICE",
    "chd_handoff_entities_facing": "DEVICE",
    "chd_follow_set_frame": "LOCK|DEVICE",
    "chd_get_follow_frame": "LOCK|COPY_WAIT",
    # chd_gpu_rings.h: neither reads the expanded list nor rewrites an array a read-back copies: the device alone
    "chd_export_ring_limits": "DEVICE",
    "chd_import_ring_limits": "DEVICE",
}
# entry points whose whole body calls another one: its CHD_ENTER is theirs
FORWARDS = {
    "chd_cell_of": "chd_cell_of_valid",
    "chd_fetch_results": "chd_fetch_results_delta",
    "chd_fetch_results_async": "chd_fetch_results_async_delta",
    "chd_fetch_wait": "chd_fetch_wait_delta",
}
# The entry points that apply rule 13 (chd_rule_no_chain: refused while a chd_begin_interest is pending, until the chd_tick that
# joins it), directly or through another rule that applies it: always, only when the begun chain includes the fan-out, or only
# with device rings.
ALWAYS, FANOUT, RINGS = "always", "fan-out only", "with device rings"
CHAIN = {
    "chd_begin_interest": ALWAYS,
    "chd_set_rings": FANOUT,
    "chd_rings_init": ALWAYS,
    "chd_rings_append": ALWAYS,
    "chd_set_channel_start_times": ALWAYS,
    "chd_follow_queries": ALWAYS,
    "chd_follow_queries_with": ALWAYS,
    "chd_get_follow": ALWAYS,
    "chd_get_follow_frame": ALWAYS,
    "chd_apply_subscriptions": ALWAYS,
    "chd_export_ring_limits": ALWAYS,
    "chd_import_ring_limits": ALWAYS,
    "chd_adjacent_broadcast": ALWAYS,
    "chd_tick_sharded": RINGS,
}
# a call of rule 13, with the flag of the engine it is guarded by (only `rings`, the engine's device rings) and fanout_only
CHAIN_CALL = r"(?:\b(\w+)\s*&&\s*)?\bchd_rule_no_chain\s*\(\s*e\s*,[^;]*?,\s*(true|false)\s*\)"
CHAIN_VARIANT = {(None, "false"): ALWAYS, (None, "true"): FANOUT, ("rings", "false"): RINGS}
# where the steps may still be written out: CHD_ENTER's implementation (chd_enter), chd_create and chd_destroy (the device);
# run_stage's capture lock and chd_update_interest_on's query-scratch lock; the waits that are not a prologue (conditional, or
# in the middle of a function), each with a comment that says when it runs
EXPLICIT = {
    "cudaSetDevice": {"chd_enter", "chd_create", "chd_destroy"},
    "e->mu": {"chd_enter", "run_stage", "chd_update_interest_on"},
    "chd_copy_wait": {"chd_enter", "chd_destroy", "chd_grow_slots", "chd_fetch_results_delta", "tick_enqueue", "chd_tick_sharded"},
    "chd_fetch_guard": {"chd_enter"},
    # the call-order state of rules 9 and 13: read by their rule functions, and set, consumed or joined by the code that starts,
    # generates, consumes or joins what it describes
    "interest_pending": {"chd_rule_no_chain", "chd_begin_interest", "tick_enqueue"},
    "pending_fanout": {"chd_rule_no_chain", "chd_begin_interest", "tick_enqueue"},
    "fw.ready": {"chd_rule_no_generated_batch", "chd_rule_batch_waiting", "follow_generate", "chd_update_interest_on"},
    "pf_q.cur": {"chd_rule_one_batch", "chd_rule_merged_batch", "chd_rule_batch_waiting", "chd_update_interest_on", "chd_follow_queries_with",
                 "chd_tick_sharded"},
}
CALLS = {
    "cudaSetDevice": r"\bcudaSetDevice\s*\(",
    "e->mu": r"\(\s*e->mu\s*\)",
    "chd_copy_wait": r"\bchd_copy_wait\s*\(\s*e\s*\)",
    "chd_fetch_guard": r"\bchd_fetch_guard\s*\(\s*e\s*,",
    "interest_pending": r"->interest_pending\b",
    "pending_fanout": r"->pending_fanout\b",
    "fw.ready": r"\b(?:e->fw|F)\.ready\b",  # (F: the engine's Follow in chd_follow.cu)
    "pf_q.cur": r"->pf_q\.cur\b",
}


def _blank(m):
    return re.sub(r"[^\n]", " ", m.group(0))


def _code(path):
    """The source with string literals and comments blanked out (offsets and line numbers kept)."""
    src = open(path).read()
    src = re.sub(r'"(?:\\.|[^"\\\n])*"', _blank, src)
    return re.sub(r"//[^\n]*|/\*.*?\*/", _blank, src, flags=re.S)


def _entry_points():
    out = set()
    for h in HEADERS:
        hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", h)).read(), flags=re.S)
        out |= {m.group(1) for m in re.finditer(r"^chd_status\s+(chd_[a-z0-9_]+)\s*\(\s*chd_engine\s*\*", hdr, flags=re.M)}
    return out


def _bodies():
    """Every function of csrc/*.cu defined at the top level: name -> body."""
    out = {}
    for path in sorted(glob.glob(os.path.join(CSRC, "*.cu"))):
        code = _code(path)
        for m in re.finditer(r"^[A-Za-z_][\w \*]*?\b(chd_[a-z0-9_]+)\s*\([^;{]*?\)\s*\{", code, flags=re.M):
            i, depth = m.end(), 1
            while depth:
                depth += {"{": 1, "}": -1}.get(code[i], 0)
                i += 1
            assert m.group(1) not in out, m.group(1)
            out[m.group(1)] = code[m.end():i - 1]
    return out


def _flags(s):
    f = {t.strip().replace("ENTRY_", "") for t in s.split("|")} - {"0"}
    return f | {"DEVICE"} if f & {"COPY_WAIT", "FETCH_GUARD"} else f


def test_every_entry_point_is_in_the_table():
    assert _entry_points() == set(NEEDS) | set(FORWARDS)


def test_each_entry_point_declares_its_needs_once():
    bodies = _bodies()
    for name, want in NEEDS.items():
        enters = re.findall(r"\bCHD_ENTER\s*\(\s*e\s*,([^;]*)\)\s*;", bodies[name])
        assert len(enters) == 1, "%s: %d CHD_ENTER" % (name, len(enters))
        assert _flags(enters[0]) == _flags(want), "%s declares %s, the table says %s" % (name, enters[0].strip(), want)
    for name, target in FORWARDS.items():
        assert re.fullmatch(r"\s*return\s+%s\s*\([^;]*\)\s*;\s*" % target, bodies[name]), name


def _chain_variants(body, via=()):
    """how a body applies rule 13: the variant of each direct call, and ALWAYS for a call of a rule in `via` (which applies it)"""
    out = {CHAIN_VARIANT.get(m.groups(), "%s && fanout_only=%s" % m.groups()) for m in re.finditer(CHAIN_CALL, body)}
    return out | {ALWAYS for name in via if re.search(r"\b%s\s*\(" % name, body)}


def test_rule_13_is_applied_where_the_chain_table_says():
    bodies = _bodies()
    via = {n for n, b in bodies.items() if n.startswith("chd_rule_") and _chain_variants(b)}
    for name in via:  # the other rules apply it whenever they get that far: their callers apply it always
        assert _chain_variants(bodies[name]) == {ALWAYS}, name
    got = {n: _chain_variants(bodies[n], via) for n in NEEDS}
    assert {n: v for n, v in got.items() if v} == {n: {v} for n, v in CHAIN.items()}


def test_the_steps_are_written_out_nowhere_else():
    found = {k: set() for k in CALLS}
    for path in sorted(glob.glob(os.path.join(CSRC, "*.cu")) + glob.glob(os.path.join(CSRC, "*.h")) + glob.glob(os.path.join(CSRC, "*.cuh"))):
        lines = _code(path).split("\n")
        for k, pat in CALLS.items():
            for no, line in enumerate(lines):
                if not re.search(pat, line) or re.match(r"\s*(cudaError_t|chd_status)\s+chd_\w+\s*\(\s*chd_engine\s*\*", line):
                    continue  # (a declaration or definition of the call itself)
                # the enclosing function: the nearest line above that starts at the first column
                head = next(l for l in reversed(lines[:no + 1]) if re.match(r"[A-Za-z_]", l))
                found[k].add(re.search(r"(\w+)\s*\(", head).group(1))
    for k in CALLS:
        assert found[k] <= EXPLICIT[k], "%s written out in %s" % (k, sorted(found[k] - EXPLICIT[k]))
