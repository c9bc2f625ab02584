# TEST INFRASTRUCTURE ONLY.  make -C oracle -f window.mk window
# Builds oracle/_ref/libdsm_refmap_window.so (the reference SurfelMap oracle of the `refmap` target of oracle/Makefile,
# same compiler and flags, with its own FusionFunctions) and, where the product library is built,
# oracle/_ref/libdsm_refmap_window_b200.so (the same node over the product adapter), each plus the hooks of
# ref_map_window.cpp.  Skipped where the reference sources are absent.
include $(dir $(abspath $(lastword $(MAKEFILE_LIST))))Makefile

window:
	@if [ -f $(REF_SRC)/surfel_map.cpp ]; then \
	  mkdir -p $(OUT) && \
	  $(MAP_CXX) $(MAP_FLAGS) -O3 -I$(HERE)shim_map -I$(HERE)shim -I$(REF_SRC) -o $(OUT)/libdsm_refmap_window.so $(HERE)ref_map_window.cpp $(HERE)ref_ff_tu.cpp && \
	  echo "built reference SurfelMap oracle with the window hooks into $(OUT)"; \
	  if [ -f $(PKG)/libdsm_b200.so ]; then \
	    $(MAP_CXX) $(MAP_FLAGS) -O2 -I$(HERE)shim_map_b200 -I$(HERE)../include -I$(HERE)shim_map -I$(HERE)shim -I$(REF_SRC) \
	      -o $(OUT)/libdsm_refmap_window_b200.so $(HERE)ref_map_window.cpp -L$(PKG) -ldsm_b200 '-Wl,-rpath,$$ORIGIN/../../densesurfelmapping_b200' && \
	    echo "built reference SurfelMap over the product adapter with the window hooks into $(OUT)"; \
	  else echo "product library not built yet: skipping libdsm_refmap_window_b200.so"; fi; \
	else echo "reference sources not present at $(REF_SRC): keeping prebuilt $(OUT)/libdsm_refmap_window*.so"; fi
.PHONY: window
