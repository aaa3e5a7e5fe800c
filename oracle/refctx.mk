# TEST INFRASTRUCTURE ONLY.  oracle/refctx.cpp (what lies ahead of every vehicle in the reference) built twice, into
# oracle/_ref/: refctx against the unmodified reference library oracle/Makefile builds (_ref/libcityflow_ref.a, so
# run `make ref` first), and refctx_lcorder from the same priority-ordered throw-away copy of the reference as
# refdump_lcorder (lc_order_patch.sh explains the one change).  Run from oracle/:  make -f refctx.mk
REF      ?= /root/reference
OUT      := _ref
CXX      ?= g++
INC      := -I$(REF)/src -I$(REF)/extern/milo -I$(REF)/extern/rapidjson/include
CXXFLAGS := -O2 -fPIC -ffp-contract=off -DRAPIDJSON_HAS_STDSTRING=1 -w
SRCS     := utility/utility utility/barrier engine/archive engine/engine flow/flow \
            roadnet/roadnet roadnet/trafficlight vehicle/router vehicle/vehicle vehicle/lanechange

all: $(OUT)/refctx $(OUT)/refctx_lcorder

$(OUT)/refctx: refctx.cpp $(OUT)/libcityflow_ref.a
	$(CXX) -std=c++11 $(CXXFLAGS) $(INC) refctx.cpp $(OUT)/libcityflow_ref.a -lpthread -o $@

$(OUT)/refctx_lcorder: refctx.cpp lc_order_patch.sh $(addprefix $(REF)/src/,$(addsuffix .cpp,$(SRCS)))
	mkdir -p $(OUT)
	set -e; tmp=$$(mktemp -d); trap 'rm -rf "$$tmp"' EXIT; cp -r $(REF)/src $$tmp/src; sh lc_order_patch.sh $$tmp/src; \
	$(CXX) -std=c++11 $(CXXFLAGS) -I$$tmp/src -I$(REF)/extern/milo -I$(REF)/extern/rapidjson/include \
	    refctx.cpp $(addprefix $$tmp/src/,$(addsuffix .cpp,$(SRCS))) -lpthread -o $@

.PHONY: all
