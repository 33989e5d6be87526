# oracle/essential.mk — checkers of the essential-matrix geometric filter (DESIGN §3.8), on top of oracle/Makefile:
#   _build/liboracle_essential.so      CPU restatement (essential_oracle.cpp; travels, built anywhere)
#   _ref/libref_geom_essential.so      the reference's own FivePointsRelativePose + ACRANSAC/ACKernelAdaptorEssential
#   _ref/dropin_essential_test         GeometricFilter_EMatrix_AC vs ImageCollectionGeometricFilter_B200::Robust_model_estimation_E
# Usage: make -f oracle/essential.mk essential-oracle | essential-ref | essential-dropin
include $(dir $(abspath $(lastword $(MAKEFILE_LIST))))Makefile

.PHONY: essential-oracle essential-ref essential-dropin
.DEFAULT_GOAL := essential-oracle
essential-oracle: $(BUILD)/liboracle_essential.so
essential-ref: $(OUT)/libref_geom_essential.so
essential-dropin: $(OUT)/dropin_essential_test

$(BUILD)/liboracle_essential.so: $(HERE)essential_oracle.cpp $(HERE)acransac_oracle.cpp
	@mkdir -p $(BUILD)
	$(CXX) -O2 -fPIC -std=c++17 -ffp-contract=off -shared -o $@ $(HERE)essential_oracle.cpp -lm

# the reference's essential-matrix TUs on top of the F/H ones (found by resolving link errors)
OMVG_GE_CC := multiview/solver_essential_five_point.cpp multiview/solver_essential_kernel.cpp multiview/essential.cpp \
              multiview/solver_essential_three_point.cpp
OMVG_GE_O  := $(patsubst %.cpp,$(OBJ)/omvg/%.o,$(OMVG_GE_CC))
$(OUT)/libref_geom_essential.so: $(HERE)ref_geom_essential_driver.cpp $(OMVG_G_O) $(OMVG_GE_O)
	@mkdir -p $(OUT)
	$(CXX) $(OPT) -std=c++11 -w -shared $(OMVG_DEF) $(OMVG_INC) $(HERE)ref_geom_essential_driver.cpp $(OMVG_G_O) $(OMVG_GE_O) -o $@ -lpthread -lm

$(OUT)/dropin_essential_test: $(HERE)dropin_essential_test.cpp $(OMVG_M_O) $(STLPLUS_O) $(OMVG_GF_O) $(OMVG_GE_O) $(B200LIB)/libomvg_b200.so \
                              $(B200LIB)/host/GeometricFilter_B200.hpp
	$(CXX) $(OPT) -std=c++11 -w $(OMVG_DEF) $(OMVG_INC) -I$(SRC)/third_party/lemon -I$(HERE)../include \
	   $(HERE)dropin_essential_test.cpp $(OMVG_M_O) $(STLPLUS_O) $(OMVG_GF_O) $(OMVG_GE_O) $(OBJ)/omvg/numeric/numeric.o \
	   -L$(B200LIB) -lomvg_b200 -Wl,-rpath,'$$ORIGIN/../../openmvg_b200' -o $@ -lpthread -lm
