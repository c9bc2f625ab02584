# TEST INFRASTRUCTURE ONLY.  make -C oracle -f clouds.mk clouds
# Builds oracle/_ref/libdsm_refmap_clouds.so: the reference SurfelMap oracle of the `refmap` target of oracle/Makefile
# (same compiler and flags) plus the hooks of ref_map_clouds.cpp.  Skipped where the reference sources are absent.
include $(dir $(abspath $(lastword $(MAKEFILE_LIST))))Makefile

clouds:
	@if [ -f $(REF_SRC)/surfel_map.cpp ]; then \
	  mkdir -p $(OUT) && \
	  $(MAP_CXX) $(MAP_FLAGS) -O3 -I$(HERE)shim_map -I$(HERE)shim -I$(REF_SRC) -o $(OUT)/libdsm_refmap_clouds.so $(HERE)ref_map_clouds.cpp $(HERE)ref_ff_tu.cpp && \
	  echo "built reference SurfelMap oracle with the cloud hooks into $(OUT)"; \
	else echo "reference sources not present at $(REF_SRC): keeping prebuilt $(OUT)/libdsm_refmap_clouds.so"; fi
.PHONY: clouds
