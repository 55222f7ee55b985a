# `make -f setvalues.mk`: the reference's fvMatrix::setValues compiled for the host against the fvMatrix shims of
# ref_harness/shim_fvm/ (test infrastructure, like `make ref` in Makefile) -> _ref/libref_setvalues.so.  Skipped where
# $(REFROOT) is absent; the library travels prebuilt.
REFROOT ?= /root/reference
CXX_REF := $(shell test -x /usr/bin/g++ && echo /usr/bin/g++ || echo g++)
CUDA_INC ?= /usr/local/cuda/include
FVMDIR = $(REFROOT)/src/finiteVolume/fvMatrices
REF_SV_FILES = $(FVMDIR)/fvMatrix/fvMatrix.H $(FVMDIR)/fvMatrix/fvMatrix.C $(FVMDIR)/fvMatrix/fvMatrixSolve.C \
            $(FVMDIR)/fvScalarMatrix/fvScalarMatrix.H $(FVMDIR)/fvScalarMatrix/fvScalarMatrix.C \
            $(REFROOT)/src/finiteVolume/finiteVolume/convectionSchemes/gaussConvectionScheme/gaussConvectionScheme.C \
            $(REFROOT)/src/finiteVolume/finiteVolume/laplacianSchemes/gaussLaplacianScheme/gaussLaplacianScheme.C \
            $(REFROOT)/src/finiteVolume/interpolation/surfaceInterpolation/surfaceInterpolationScheme/surfaceInterpolationScheme.C \
            $(REFROOT)/src/finiteVolume/finiteVolume/ddtSchemes/ddtScheme/ddtScheme.C \
            $(REFROOT)/src/finiteVolume/finiteVolume/ddtSchemes/EulerDdtScheme/EulerDdtScheme.C
REF_SV_OUT = _ref/libref_setvalues.so

ref:
	@if [ -d "$(FVMDIR)" ]; then $(MAKE) -f setvalues.mk $(REF_SV_OUT); else echo "reference tree not present: keeping prebuilt $(REF_SV_OUT) if any"; fi

$(REF_SV_OUT): ref_harness/harness_setvalues.cpp ref_harness/harness_fvm.cpp ref_harness/shim_fvm/fvm_shim.h $(REF_SV_FILES)
	mkdir -p _ref/inc_sv
	for f in $(REF_SV_FILES); do ln -sf $$f _ref/inc_sv/; done
	$(CXX_REF) -O2 -fPIC -std=c++17 -ffp-contract=off -fno-fast-math -w \
	    -DTHRUST_DEVICE_SYSTEM=THRUST_DEVICE_SYSTEM_CPP -DTHRUST_HOST_SYSTEM=THRUST_HOST_SYSTEM_CPP \
	    -DCCCL_IGNORE_DEPRECATED_CPP_DIALECT \
	    -iquote _ref/inc_sv -I ref_harness/shim_fvm -I ref_harness -I _ref/inc_sv -isystem $(CUDA_INC) \
	    -shared -o $@ ref_harness/harness_setvalues.cpp
	rm -rf _ref/inc_sv

.PHONY: ref
