import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
import dial_mpc_b200.envs as E
from dial_mpc_b200 import random as drandom
from dial_mpc_b200.core.dial_config import DialConfig
from dial_mpc_b200.core.dial_core import MBDPI
name = sys.argv[1]; N = int(sys.argv[2]); Hs = int(sys.argv[3]); Hn = int(sys.argv[4])
if name == 'unitree_go2_walk': ecfg = E.UnitreeGo2EnvConfig(default_vx=0.8, ramp_up_time=1.0)
elif name == 'unitree_go2_seq_jump': ecfg = E.UnitreeGo2SeqJumpEnvConfig(pose_target_sequence=np.array([[0,0,0.27],[0.4,0,0.27],[0.8,0,0.27],[1.2,0,0.27],[1.6,0,0.27]]), yaw_target_sequence=np.zeros(5))
elif name == 'allegro_reorient': ecfg = E.AllegroReorientEnvConfig(dt=0.02, timestep=0.005, leg_control='position')
else: ecfg = E.UnitreeH1WalkEnvConfig(default_vx=2.0, ramp_up_time=3.0)
env = E.get_environment(name, config=ecfg)
mb = MBDPI(DialConfig(env_name=name, Nsample=N, Hsample=Hs, Hnode=Hn, temp_sample=0.05), env)
st = env.reset(drandom.PRNGKey(0))
for _ in range(0 if name == 'allegro_reorient' else 10): st = env.step(st, torch.zeros(mb.nu, device=mb.device))
Y = torch.zeros(Hn + 1, mb.nu, device=mb.device); key = drandom.PRNGKey(1)
for i in range(3): mb.plan.reverse_rollout(st, None, key, Y, mb.sigma_control, mb._rews_local)
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for i in range(20): mb.plan.reverse_rollout(st, None, key, Y, mb.sigma_control, mb._rews_local)
e1.record(); torch.cuda.synchronize()
ms = e0.elapsed_time(e1) / 20
print(f"{name} N={N} Hs={Hs} WPC={os.environ.get('DIAL_WPC','auto')}: rollout kernel {ms:.3f} ms -> {N*Hs/ms*1e3:.3e} sample-steps/s  rews {float(mb._rews_local.mean()):.5f}")
