// The built-in SafetyCarButton1Gymnasium-v0 struct as a plugin: its collects must be bit-identical to the built-in kind's.
#include "envs.cuh"
using UserEnv = fsrl::Env<fsrl::ENV_CAR_BUTTON1>;
