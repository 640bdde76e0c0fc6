# The compiler and flags of every CUDA object of the project: the library (Makefile) and the env plugins
# (`make plugin`, fsrl_b200.envs.build_device_env).  One definition, so a plugin of a built-in env struct
# compiles to the same kernels as the library's instantiation of it.
NVCC ?= /usr/local/cuda/bin/nvcc
ARCH := -gencode arch=compute_90a,code=sm_90a
NVCCFLAGS ?= -O3 -std=c++17 -lineinfo $(ARCH) -Xcompiler -fPIC -Xptxas -v --expt-relaxed-constexpr
# extra flags for instrumented builds, e.g. EXTRA_NVCCFLAGS=-DFSRL_PPO_CHUNK_STAMPS (csrc/ppo_persist.cu)
NVCCFLAGS += $(EXTRA_NVCCFLAGS)
