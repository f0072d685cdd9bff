"""nvidia-smi sampling for the benchmark tools: the card name and power limit, and the SM clock and active throttle reasons during a timed window."""
import statistics, subprocess, threading, time


class SmiSampler:
    """nvidia-smi samples (SM clock MHz, active throttle reasons) every 0.2 s while active; card name and power limit read once"""

    Q = "clocks.sm,clocks_throttle_reasons.active"

    def __init__(self):
        self.samples, self.stop = [], threading.Event()
        try:
            self.card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
        except (OSError, subprocess.TimeoutExpired):
            self.card = "unknown"

    def _run(self):
        while not self.stop.is_set():
            try:
                out = subprocess.run(["nvidia-smi", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits", "-i", "0"], capture_output=True, text=True, timeout=10).stdout
                clk, thr = [t.strip() for t in out.strip().split(",")]
                self.samples.append((float(clk), thr))
            except (OSError, ValueError, subprocess.TimeoutExpired):
                pass
            time.sleep(0.2)

    def __enter__(self):
        self.t = threading.Thread(target=self._run, daemon=True); self.t.start(); return self

    def __exit__(self, *a):
        self.stop.set(); self.t.join()

    def summary(self):
        return {"card": self.card, "sm_clock_mhz_median": statistics.median([c for c, _ in self.samples]) if self.samples else None,
                "throttle_reasons": sorted({t for _, t in self.samples})}
