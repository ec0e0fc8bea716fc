"""Diagnostic: is the config-2 launch (256 chains, D=1024, L=10, S=1000, in-kernel Philox) power-bound?

Times the launch two ways, as isolated launches (event pair, synchronise and 20 ms of idle after each) and as launches
queued back to back (as bench.py issues them), and reads NVML around both: total energy before and after, and every
10 ms the power draw, SM clock, clock-event reasons and temperature.  An idle second first gives the card's idle power.
If the queued run drew power at the enforced limit, with sw_power_cap set and the SM clock below its maximum, the time
it loses against isolated launches would be power; otherwise it is the kernel's own stalls.  Prints one JSON line per
run, headed by the card's name, power limit and maximum SM clock."""
import json, os, sys, threading, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import pynvml as nv
import torch
from hamiltorch_b200 import engine, targets as T

REASONS = (('hw_slowdown', 'nvmlClocksEventReasonHwSlowdown'), ('hw_power_brake', 'nvmlClocksEventReasonHwPowerBrakeSlowdown'),
           ('sw_power_cap', 'nvmlClocksEventReasonSwPowerCap'), ('sw_thermal', 'nvmlClocksEventReasonSwThermalSlowdown'),
           ('hw_thermal', 'nvmlClocksEventReasonHwThermalSlowdown'))

nv.nvmlInit()
vis = os.environ.get('CUDA_VISIBLE_DEVICES', '0').split(',')[0].strip()
h = nv.nvmlDeviceGetHandleByIndex(int(vis) if vis.isdigit() else 0)
dev = torch.device('cuda', 0)
tgt = engine.NativeTarget(T.GaussianIso(1024), dev)
q0 = (0.1 * torch.randn(256, 1024, generator=torch.Generator().manual_seed(0))).to(dev)
out = torch.empty((256, 1000, 1024), dtype=torch.float32, device=dev)


def launch(k):
    return engine.hmc_run(tgt, q0, 1000, 10, 0.05, seed=k, out=out, device=dev)


def med(v):
    return sorted(v)[len(v) // 2]


class Poll:
    def __init__(self):
        self.stop, self.power, self.clock, self.temp, self.reasons = False, [], [], [], {}
        self.thread = threading.Thread(target=self.loop, daemon=True)

    def loop(self):
        while not self.stop:
            self.power.append(nv.nvmlDeviceGetPowerUsage(h) / 1e3)
            self.clock.append(nv.nvmlDeviceGetClockInfo(h, nv.NVML_CLOCK_SM))
            self.temp.append(nv.nvmlDeviceGetTemperature(h, nv.NVML_TEMPERATURE_GPU))
            r = nv.nvmlDeviceGetCurrentClocksEventReasons(h)
            for name, const in REASONS:
                if r & getattr(nv, const):
                    self.reasons[name] = self.reasons.get(name, 0) + 1
            time.sleep(0.01)

    def __enter__(self):
        torch.cuda.synchronize()
        self.e0, self.t0 = nv.nvmlDeviceGetTotalEnergyConsumption(h), time.time()
        self.thread.start()
        return self

    def __exit__(self, *exc):
        torch.cuda.synchronize()
        self.stop = True
        self.thread.join()
        self.wall = time.time() - self.t0
        self.joules = (nv.nvmlDeviceGetTotalEnergyConsumption(h) - self.e0) / 1e3

    def fields(self):
        return dict(wall_s=round(self.wall, 3), energy_j=round(self.joules, 1), power_w_median=med(self.power),
                    power_w_max=max(self.power), sm_mhz_median=med(self.clock), sm_mhz_min=min(self.clock),
                    temp_c_max=max(self.temp), reason_polls=self.reasons, polls=len(self.power))


def run(mode, n):
    times = []
    with Poll() as p:
        if mode == 'queued':
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for k in range(n):
                launch(k)
            e1.record()
            torch.cuda.synchronize()
            times = [e0.elapsed_time(e1) / n]
        else:
            for k in range(n):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                launch(k)
                e1.record()
                torch.cuda.synchronize()
                times.append(e0.elapsed_time(e1))
                time.sleep(0.02)
    return dict(mode=mode, launches=n, ms_per_launch=med(times), mj_per_iteration_incl_idle=p.joules / (n * 1000) * 1e3,
                **p.fields())


print(json.dumps(dict(card=nv.nvmlDeviceGetName(h), power_limit_w=nv.nvmlDeviceGetEnforcedPowerLimit(h) / 1e3,
                      max_sm_mhz=nv.nvmlDeviceGetMaxClockInfo(h, nv.NVML_CLOCK_SM))))
with Poll() as idle:
    time.sleep(1.0)
print(json.dumps(dict(mode='idle', **idle.fields())))
for k in range(30):
    launch(k)
for rep in range(2):
    print(json.dumps(run('isolated', 60)))
    print(json.dumps(run('queued', 1500)))
