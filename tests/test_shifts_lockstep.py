"""The lockstep shift solver (calculate_shifts_many) on the CPU, with the oracle's streams as the matcher backend and an
executor that answers every round request by request: per-event results equal calculate_shifts run on each job alone,
and the number of rounds is the largest per-job request count, not their sum."""
import numpy as np
import pytest

from sushi_b200.events import ScriptEvent
from sushi_b200.grouping import prepare_search_groups
from sushi_b200.shifts import _answer_alone, calculate_shifts, calculate_shifts_many
from tests.helpers import oracle_stream_from_pcm
from tests.test_shifts_host import scenario_inputs


def per_request(batch):
    return [_answer_alone(src, dst, req) for src, dst, req in batch]


def outcome(events):
    return [(e.shift, e.diff, e._link.source_index if e.linked else -1) for e in events]


@pytest.fixture(scope='module')
def scenarios(golden_shifts):
    out = {}
    for name in ('const', 'jump', 'rewind'):
        src_pcm, dst_pcm, ev, params = scenario_inputs(golden_shifts, name)
        out[name] = (oracle_stream_from_pcm(src_pcm, 12000, 1, 12000, 'uint8'),
                     oracle_stream_from_pcm(dst_pcm, 12000, 1, 12000, 'uint8'), ev, params)
    # the const scenario against the first 30 % of its destination: the later groups lie past the end of the audio
    src_pcm, dst_pcm, ev, params = scenario_inputs(golden_shifts, 'const')
    out['short_dst'] = (out['const'][0], oracle_stream_from_pcm(dst_pcm[:int(len(dst_pcm) * 0.3)], 12000, 1, 12000, 'uint8'), ev, params)
    return out


def make_job(scenarios, name, dst=None):
    src, d, ev, params = scenarios[name]
    events = [ScriptEvent(i, float(a), float(b)) for i, (a, b) in enumerate(ev)]
    groups = prepare_search_groups(events, src.duration_seconds, [], 0.417, 0.417)
    return events, (src, dst or d, groups), params


def test_lockstep_equals_per_job_solver_and_rounds_are_the_maximum(scenarios):
    params = scenarios['const'][3]
    window, max_window, rewind = float(params[0]), float(params[1]), int(params[2])
    for name in ('jump', 'rewind', 'short_dst'):
        assert tuple(scenarios[name][3]) == tuple(params)          # one solver setting for every job
    shared_dst = scenarios['jump'][1]
    specs = [('const', None), ('jump', None), ('rewind', None), ('short_dst', None),
             ('const', shared_dst), ('jump', shared_dst),             # two jobs sharing a destination stream
             ('empty', None)]                                         # a job without groups

    def build():
        jobs, events = [], []
        for name, dst in specs:
            if name == 'empty':
                events.append([])
                jobs.append((scenarios['const'][0], scenarios['const'][1], []))
                continue
            ev, job, _ = make_job(scenarios, name, dst)
            events.append(ev)
            jobs.append(job)
        return jobs, events

    # each job alone: the sequential solver, and its request count through the lockstep driver
    alone, counts = [], []
    jobs, events = build()
    for job, ev in zip(jobs, events):
        calculate_shifts(job[0], job[1], job[2], window, max_window, rewind)
        alone.append(outcome(ev))
    jobs, events = build()
    for job in jobs:
        counts.append(calculate_shifts_many([job], window, max_window, rewind, executor=per_request))
    assert counts[-1] == 0 and max(counts) > 0
    # all jobs together
    jobs, events = build()
    rounds = calculate_shifts_many(jobs, window, max_window, rewind, executor=per_request)
    assert rounds == max(counts) < sum(counts)
    for k, ev in enumerate(events):
        assert outcome(ev) == alone[k], specs[k]
    # the short destination really ends early: the last groups are left without a shift and linked instead
    short = events[specs.index(('short_dst', None))]
    assert short[-1].linked


def test_lockstep_answers_probes_in_order(scenarios):
    """The executor sees one request per waiting job per round, in job order, and probe triples as three searches."""
    params = scenarios['rewind'][3]
    seen = []

    def spy(batch):
        seen.append([req[0] for _, _, req in batch])
        for _, _, req in batch:
            assert req[0] in ('probe', 'find')
            if req[0] == 'probe':
                assert len(req[1]) == 3
        return per_request(batch)

    jobs = [make_job(scenarios, 'rewind')[1], make_job(scenarios, 'jump')[1]]
    calculate_shifts_many(jobs, float(params[0]), float(params[1]), int(params[2]), executor=spy)
    assert seen and all(1 <= len(r) <= 2 for r in seen) and 'probe' in np.concatenate(seen)
