"""Entry point of a FRESH process (tests/test_host_mock_engine_cpu.py spawns it): load the CPU mock of the engine entry
points with RTLD_GLOBAL first, so that libmkhost's mksnap_* references bind to it, then run one scenario.
    python -m tests.mock_engine.run <mock.so> <scenario> <tmpdir>"""
import sys

from tests.mock_engine import load_for_child


def main():
    mock_path, scenario, tmp = sys.argv[1:4]
    mock = load_for_child(mock_path, host=True)
    from tests.mock_engine import scenarios
    getattr(scenarios, scenario)(scenarios.MockEngineFactory(mock), tmp)
    print("SCENARIO-OK", scenario)


if __name__ == "__main__":
    main()
