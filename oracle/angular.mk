# oracle/angular.mk — checkers of the angular essential-matrix geometric filters (`-g a` / `-g u`, DESIGN §3.10), on top
# of oracle/Makefile and oracle/essential.mk:
#   _build/liboracle_angular.so        CPU restatement (angular_oracle.cpp; travels, built anywhere)
#   _ref/libref_geom_angular.so        the reference's own solvers, AngularError, ACRANSAC/ACKernelAdaptor_AngularRadianError
#                                      and RelativePoseFromEssential
#   _ref/dropin_angular_test           GeometricFilter_ESphericalMatrix_AC_Angular<false | true> vs
#                                      ImageCollectionGeometricFilter_B200::Robust_model_estimation_EAngular / _EUpright
# Usage: make -f oracle/angular.mk angular-oracle | angular-ref | angular-dropin
include $(dir $(abspath $(lastword $(MAKEFILE_LIST))))essential.mk

.PHONY: angular-oracle angular-ref angular-dropin
.DEFAULT_GOAL := angular-oracle
angular-oracle: $(BUILD)/liboracle_angular.so
angular-ref: $(OUT)/libref_geom_angular.so
angular-dropin: $(OUT)/dropin_angular_test

$(BUILD)/liboracle_angular.so: $(HERE)angular_oracle.cpp $(HERE)acransac_oracle.cpp
	@mkdir -p $(BUILD)
	$(CXX) -O2 -fPIC -std=c++17 -ffp-contract=off -shared -o $@ $(HERE)angular_oracle.cpp -lm

# the reference's angular TUs on top of the essential ones (found by resolving link errors)
OMVG_GA_CC := multiview/solver_essential_eight_point.cpp multiview/motion_from_essential.cpp multiview/triangulation.cpp
OMVG_GA_O  := $(patsubst %.cpp,$(OBJ)/omvg/%.o,$(OMVG_GA_CC))
$(OUT)/libref_geom_angular.so: $(HERE)ref_geom_angular_driver.cpp $(OMVG_G_O) $(OMVG_GE_O) $(OMVG_GA_O)
	@mkdir -p $(OUT)
	$(CXX) $(OPT) -std=c++11 -w -shared -Wl,--no-undefined $(OMVG_DEF) $(OMVG_INC) $(HERE)ref_geom_angular_driver.cpp $(OMVG_G_O) $(OMVG_GE_O) $(OMVG_GA_O) -o $@ -lpthread -lm

$(OUT)/dropin_angular_test: $(HERE)dropin_angular_test.cpp $(OMVG_M_O) $(STLPLUS_O) $(OMVG_GF_O) $(OMVG_GE_O) $(OMVG_GA_O) $(B200LIB)/libomvg_b200.so \
                            $(B200LIB)/host/GeometricFilter_B200.hpp
	$(CXX) $(OPT) -std=c++11 -w $(OMVG_DEF) $(OMVG_INC) -I$(SRC)/third_party/lemon -I$(HERE)../include \
	   $(HERE)dropin_angular_test.cpp $(OMVG_M_O) $(STLPLUS_O) $(OMVG_GF_O) $(OMVG_GE_O) $(OMVG_GA_O) $(OBJ)/omvg/numeric/numeric.o \
	   -L$(B200LIB) -lomvg_b200 -Wl,-rpath,'$$ORIGIN/../../openmvg_b200' -o $@ -lpthread -lm
