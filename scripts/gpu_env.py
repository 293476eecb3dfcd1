"""The card a measurement ran on, read with nvidia-smi: its name and power limit, and its SM clock sampled while a timed
loop runs.  Scripts record these beside their numbers."""
import subprocess
import threading


def smi(query):
    """the first line of `nvidia-smi --query-gpu=<query>`, or None if nvidia-smi cannot be read"""
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={query}", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30)
        return r.stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        return None


def gpu_name_and_power():
    """'<name>, <power limit>' of the first card"""
    return smi("name,power.limit")


class ClockSampler:
    """SM clock (MHz) sampled by nvidia-smi every 0.2 s while active"""

    def __init__(self):
        self.samples, self._stop = [], threading.Event()

    def __enter__(self):
        self._stop.clear()
        self._t = threading.Thread(target=self._run, daemon=True)
        self._t.start()
        return self

    def _run(self):
        while not self._stop.wait(0.2):
            try:
                self.samples.append(float(smi("clocks.sm").split()[0]))
            except (AttributeError, ValueError, IndexError):
                pass

    def __exit__(self, *exc):
        self._stop.set()
        self._t.join()
