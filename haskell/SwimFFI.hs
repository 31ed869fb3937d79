{-# LANGUAGE ForeignFunctionInterface #-}
{-# LANGUAGE RecordWildCards          #-}
-- | Binding of libswim_b200.so (include/swim.h) for the reference code base (jpfuentes2/swim).
--
-- NOT COMPILED IN THIS REPOSITORY'S IMAGE: there is no ghc / stack / cabal here (see INTEGRATION.md).
-- The struct layouts below are the ones tests/test_abi.py checks against the C header
-- (sizes: swim_config_t 64, swim_member_t 24, swim_message_t 48, swim_gossip_t 56, swim_event_t 64).
-- The same entry points are exercised from Python ctypes (swim_b200/_lib.py, swim_b200/core.py).
--
-- Drop this module into src/, add `extra-libraries: swim_b200` to swim.cabal, and Core.hs's functions
-- can delegate to the accelerated implementation (section 3 of INTEGRATION.md).
module SwimFFI
  ( Sim, CConfig(..), CMember(..), CMessage(..), CGossip(..), CJoin(..)
  , defaultConfig, simCreate, simDestroy, simSetView, simStep, simDigest, simMismatches
  , getMembers, setMembers, kRandomMembers, removeDeadNodes, nextSeqNo, nextIncarnation
  , suspectNode, deadNode, aliveNode, handleMessage, broadcast
  , msgPing, msgIndirectPing, msgAck, msgSuspect, msgAlive, msgDead
    -- raw imports of the bulk / codec / replay entry points (marshalled by the caller)
  , c_simSetRound, c_simSave, c_simLoad, c_simSetParams, c_simInject, c_simGetArray, c_simSetArray, c_simCounters, c_simObserve, c_simExportRound
  , c_simInjectDatagram, c_getBroadcasts, c_takeBroadcasts, c_tickTimers, c_envEncode, c_envDecode, simCounters
    -- bulk membership edits between steps: removeDeadNodes / addNewMember on every store at once
  , c_simRemoveDeadNodes, c_simAddMembers
    -- seed joins between steps: Join(joinHosts) for many processes at once
  , simJoin, joinFresh, c_simJoin
    -- graceful leaves between steps: memberlist's Leave for many processes at once
  , simLeave, c_simLeave
  ) where

import Control.Monad (when)
import Data.Int (Int32, Int64)
import Data.Word (Word16, Word32, Word64, Word8)
import Foreign
import Foreign.C.String (CString, peekCString)
import Foreign.C.Types (CInt (..), CSize (..))

data SwimSim
type Sim = Ptr SwimSim

-- MsgType (Types.hs:159-167)
msgPing, msgIndirectPing, msgAck, msgSuspect, msgAlive, msgDead :: Word8
msgPing = 0; msgIndirectPing = 1; msgAck = 2; msgSuspect = 3; msgAlive = 4; msgDead = 5

-- | swim_config_t (Config, Types.hs:46-51, plus the simulator's knobs)
data CConfig = CConfig
  { cfgAbiVersion, cfgNNodes, cfgViewCap, cfgKIndirect, cfgFanout, cfgPbCap, cfgSuspicionRounds
  , cfgRetransmit, cfgLossPpm, cfgFlags :: !Word32
  , cfgSeed :: !Word64
  , cfgRank, cfgWorld :: !Word32
  , cfgDevice :: !Int32
  , cfgBasePort :: !Word32
  , cfgChurnPpm, cfgRejoinMin, cfgRejoinMax, cfgProbesPerRound, cfgSuspicionMax :: !Word32 }

instance Storable CConfig where
  sizeOf _ = 88
  alignment _ = 8
  peek p = CConfig <$> peekByteOff p 0 <*> peekByteOff p 4 <*> peekByteOff p 8 <*> peekByteOff p 12
                   <*> peekByteOff p 16 <*> peekByteOff p 20 <*> peekByteOff p 24 <*> peekByteOff p 28
                   <*> peekByteOff p 32 <*> peekByteOff p 36 <*> peekByteOff p 40 <*> peekByteOff p 48
                   <*> peekByteOff p 52 <*> peekByteOff p 56 <*> peekByteOff p 60 <*> peekByteOff p 64
                   <*> peekByteOff p 68 <*> peekByteOff p 72 <*> peekByteOff p 76 <*> peekByteOff p 80
  poke p CConfig{..} = do
    fillBytes p 0 88
    pokeByteOff p 0 cfgAbiVersion; pokeByteOff p 4 cfgNNodes; pokeByteOff p 8 cfgViewCap
    pokeByteOff p 12 cfgKIndirect; pokeByteOff p 16 cfgFanout; pokeByteOff p 20 cfgPbCap
    pokeByteOff p 24 cfgSuspicionRounds; pokeByteOff p 28 cfgRetransmit; pokeByteOff p 32 cfgLossPpm
    pokeByteOff p 36 cfgFlags; pokeByteOff p 40 cfgSeed; pokeByteOff p 48 cfgRank; pokeByteOff p 52 cfgWorld
    pokeByteOff p 56 cfgDevice; pokeByteOff p 60 cfgBasePort; pokeByteOff p 64 cfgChurnPpm
    pokeByteOff p 68 cfgRejoinMin; pokeByteOff p 72 cfgRejoinMax; pokeByteOff p 76 cfgProbesPerRound
    pokeByteOff p 80 cfgSuspicionMax

-- | swim_member_t (Member, Types.hs:62-68; name -> id, memberHostNew -> addr/port, lastChange -> round)
data CMember = CMember
  { mId, mAddr :: !Word32, mPort :: !Word16, mLiveness, mTimer :: !Word8, mIncarnation :: !Word32
  , mLastChange :: !Word64 } deriving (Eq, Show)

instance Storable CMember where
  sizeOf _ = 24
  alignment _ = 8
  peek p = CMember <$> peekByteOff p 0 <*> peekByteOff p 4 <*> peekByteOff p 8 <*> peekByteOff p 10
                   <*> peekByteOff p 11 <*> peekByteOff p 12 <*> peekByteOff p 16
  poke p CMember{..} = do
    pokeByteOff p 0 mId; pokeByteOff p 4 mAddr; pokeByteOff p 8 mPort; pokeByteOff p 10 mLiveness
    pokeByteOff p 11 mTimer; pokeByteOff p 12 mIncarnation; pokeByteOff p 16 mLastChange

-- | swim_message_t (Message, Types.hs:122-145), tagged by kind = MsgType index
data CMessage = CMessage
  { msgKind, msgPayloadLen :: !Word8, msgPort :: !Word16, msgSeqNo, msgNode, msgTarget :: !Word32
  , msgIncarnation :: !Int64, msgDeadFrom :: !Word32 } deriving (Eq, Show)

instance Storable CMessage where
  sizeOf _ = 48
  alignment _ = 8
  peek p = CMessage <$> peekByteOff p 0 <*> peekByteOff p 1 <*> peekByteOff p 2 <*> peekByteOff p 4
                    <*> peekByteOff p 8 <*> peekByteOff p 12 <*> peekByteOff p 16 <*> peekByteOff p 24
  poke p CMessage{..} = do
    fillBytes p 0 48
    pokeByteOff p 0 msgKind; pokeByteOff p 1 msgPayloadLen; pokeByteOff p 2 msgPort; pokeByteOff p 4 msgSeqNo
    pokeByteOff p 8 msgNode; pokeByteOff p 12 msgTarget; pokeByteOff p 16 msgIncarnation; pokeByteOff p 24 msgDeadFrom

-- | swim_gossip_t (Gossip = Direct Message SockAddr | Broadcast Message, Types.hs:42-44)
data CGossip = CGossip { gIsDirect :: !Word8, gDestPort :: !Word16, gDestAddr :: !Word32, gMsg :: !CMessage }
  deriving (Eq, Show)

instance Storable CGossip where
  sizeOf _ = 56
  alignment _ = 8
  peek p = CGossip <$> peekByteOff p 0 <*> peekByteOff p 2 <*> peekByteOff p 4 <*> peek (p `plusPtr` 8)
  poke p CGossip{..} = do
    fillBytes p 0 56
    pokeByteOff p 0 gIsDirect; pokeByteOff p 2 gDestPort; pokeByteOff p 4 gDestAddr; poke (p `plusPtr` 8) gMsg

-- | swim_join_t: one joiner and one of its join hosts (Config.joinHosts, Types.hs:47)
data CJoin = CJoin { jNode, jSeed :: !Word32 } deriving (Eq, Show)

instance Storable CJoin where
  sizeOf _ = 8
  alignment _ = 4
  peek p = CJoin <$> peekByteOff p 0 <*> peekByteOff p 4
  poke p CJoin{..} = pokeByteOff p 0 jNode >> pokeByteOff p 4 jSeed

foreign import ccall unsafe "swim_config_default"    c_configDefault :: Ptr CConfig -> IO CInt
foreign import ccall safe   "swim_sim_create"        c_simCreate     :: Ptr CConfig -> Ptr Sim -> IO CInt
foreign import ccall safe   "swim_sim_destroy"       simDestroy      :: Sim -> IO ()
foreign import ccall unsafe "swim_last_error"        c_lastError     :: Sim -> IO CString
foreign import ccall safe   "swim_sim_set_view"      c_simSetView    :: Sim -> Ptr Word32 -> IO CInt
foreign import ccall safe   "swim_sim_step"          c_simStep       :: Sim -> Word32 -> IO CInt
foreign import ccall safe   "swim_sim_set_round"     c_simSetRound   :: Sim -> Word32 -> IO CInt
foreign import ccall safe   "swim_sim_save"          c_simSave       :: Sim -> IO CInt
foreign import ccall safe   "swim_sim_load"          c_simLoad       :: Sim -> IO CInt
foreign import ccall safe   "swim_sim_set_params"    c_simSetParams  :: Sim -> Ptr CConfig -> IO CInt
foreign import ccall safe   "swim_sim_digest"        c_simDigest     :: Sim -> Ptr Word64 -> IO CInt
foreign import ccall safe   "swim_sim_mismatches"    c_simMismatches :: Sim -> Ptr Word64 -> IO CInt
foreign import ccall safe   "swim_get_members"       c_getMembers    :: Sim -> Word32 -> Ptr CMember -> CSize -> Ptr CSize -> IO CInt
foreign import ccall safe   "swim_set_members"       c_setMembers    :: Sim -> Word32 -> Ptr CMember -> CSize -> IO CInt
foreign import ccall safe   "swim_k_random_members"  c_kRandom       :: Sim -> Word32 -> Word32 -> Ptr CMember -> CSize -> Ptr CMember -> CSize -> Ptr CSize -> IO CInt
foreign import ccall safe   "swim_remove_dead_nodes" c_removeDead    :: Sim -> Word32 -> IO CInt
foreign import ccall safe   "swim_next_seqno"        c_nextSeqNo     :: Sim -> Word32 -> Ptr Word32 -> IO CInt
foreign import ccall safe   "swim_next_incarnation"  c_nextInc       :: Sim -> Word32 -> Ptr Word32 -> IO CInt
foreign import ccall safe   "swim_suspect_node"      c_suspectNode   :: Sim -> Word32 -> Ptr CMessage -> Ptr CMessage -> Ptr CInt -> IO CInt
foreign import ccall safe   "swim_dead_node"         c_deadNode      :: Sim -> Word32 -> Ptr CMessage -> Ptr CMessage -> Ptr CInt -> IO CInt
foreign import ccall safe   "swim_alive_node"        c_aliveNode     :: Sim -> Word32 -> Ptr CMessage -> Ptr CMessage -> Ptr CInt -> IO CInt
foreign import ccall safe   "swim_handle_message"    c_handleMessage :: Sim -> Word32 -> Word32 -> Word16 -> Ptr CMessage -> Ptr CGossip -> CSize -> Ptr CSize -> IO CInt
foreign import ccall safe   "swim_broadcast"         c_broadcast     :: Sim -> Word32 -> Ptr CMessage -> IO CInt

-- bulk state access, datagram export/replay and the codec (Types.hs:96-119,151-155)
foreign import ccall safe   "swim_sim_inject"          c_simInject         :: Sim -> Ptr () -> CSize -> IO CInt
foreign import ccall safe   "swim_sim_get_array"       c_simGetArray       :: Sim -> CInt -> Ptr () -> CSize -> IO CInt
foreign import ccall safe   "swim_sim_set_array"       c_simSetArray       :: Sim -> CInt -> Ptr () -> CSize -> IO CInt
foreign import ccall safe   "swim_sim_counters"        c_simCounters       :: Sim -> Ptr Word64 -> CSize -> IO CInt
foreign import ccall safe   "swim_sim_observe"         c_simObserve        :: Sim -> Ptr Word64 -> CSize -> Ptr Word64 -> Ptr Word64 -> IO CInt
foreign import ccall safe   "swim_sim_export_round"    c_simExportRound    :: Sim -> Ptr Word8 -> CSize -> Ptr () -> CSize -> Ptr CSize -> Ptr CSize -> IO CInt
foreign import ccall safe   "swim_sim_inject_datagram" c_simInjectDatagram :: Sim -> Word32 -> Word32 -> Ptr Word8 -> CSize -> IO CInt
foreign import ccall safe   "swim_get_broadcasts"      c_getBroadcasts     :: Sim -> Word32 -> Ptr CMessage -> CSize -> Ptr CSize -> IO CInt
foreign import ccall safe   "swim_take_broadcasts"     c_takeBroadcasts    :: Sim -> Word32 -> Ptr CMessage -> CSize -> Ptr CSize -> IO CInt
foreign import ccall safe   "swim_tick_timers"         c_tickTimers        :: Sim -> Word32 -> Ptr Word32 -> IO CInt
-- removeDeadNodes (Core.hs:65-67) with a minimum age, and addNewMember (Core.hs:206-216) over an array of
-- swim_member_add_t {observer, member, incarnation, _pad :: Word32}; single shard, between steps
foreign import ccall safe   "swim_sim_remove_dead_nodes" c_simRemoveDeadNodes :: Sim -> Word32 -> Ptr Word64 -> IO CInt
foreign import ccall safe   "swim_sim_add_members"     c_simAddMembers     :: Sim -> Ptr Word32 -> CSize -> Ptr Word64 -> Ptr Word64 -> IO CInt
-- push-pull anti-entropy between steps (memberlist; joinHosts, Types.hs:47, completed): exchanges, inserted, full
foreign import ccall safe   "swim_sim_push_pull"       c_simPushPull       :: Sim -> Ptr Word64 -> Ptr Word64 -> Ptr Word64 -> IO CInt
-- seed joins between steps (Config.joinHosts, Types.hs:47; Util.hs:46): pairs, count, flags; exchanges, inserted, full
foreign import ccall safe   "swim_sim_join"            c_simJoin           :: Sim -> Ptr CJoin -> CSize -> Word32 -> Ptr Word64 -> Ptr Word64 -> Ptr Word64 -> IO CInt
-- graceful leaves between steps (memberlist's Leave; the reference has none): ids, count; left, delivered
foreign import ccall safe   "swim_sim_leave"           c_simLeave          :: Sim -> Ptr Word32 -> CSize -> Ptr Word64 -> Ptr Word64 -> IO CInt
-- the view graph generated on the device (kind = SWIM_TOPO_*, degree, seed) and installed as by swim_sim_set_view_device
foreign import ccall safe   "swim_sim_generate_view"   c_simGenerateView   :: Sim -> CInt -> Word32 -> Word64 -> IO CInt
foreign import ccall unsafe "swim_envelope_encode"     c_envEncode         :: Ptr () -> CSize -> Ptr Word8 -> CSize -> Ptr CSize -> IO CInt
foreign import ccall unsafe "swim_envelope_decode"     c_envDecode         :: Ptr Word8 -> CSize -> Ptr () -> CSize -> Ptr CSize -> IO CInt

-- | `Left err` / `fail` of the reference (Types.hs:33, Core.hs:87,274): every call returns 0 or SWIM_E*.
orFail :: Sim -> CInt -> IO ()
orFail sim rc = when (rc /= 0) $ c_lastError sim >>= peekCString >>= fail

defaultConfig :: IO CConfig                                         -- parseConfig (Util.hs:44-50)
defaultConfig = alloca $ \p -> c_configDefault p >>= orFail nullPtr >> peek p

simCreate :: CConfig -> IO Sim                                      -- configure / makeStore (Util.hs:76-107)
simCreate cfg = with cfg $ \pc -> alloca $ \ps -> c_simCreate pc ps >>= orFail nullPtr >> peek ps

simSetView :: Sim -> [Word32] -> IO ()                              -- bulk `swapTVar storeMembers` (Spec.hs:101)
simSetView sim ids = withArray ids $ \p -> c_simSetView sim p >>= orFail sim

simStep :: Sim -> Word32 -> IO ()                                   -- failureDetector + receiver + disseminate for all nodes
simStep sim n = c_simStep sim n >>= orFail sim

simDigest, simMismatches :: Sim -> IO Word64
simDigest sim = alloca $ \p -> c_simDigest sim p >>= orFail sim >> peek p
simMismatches sim = alloca $ \p -> c_simMismatches sim p >>= orFail sim >> peek p

simCounters :: Sim -> IO [Word64]                                   -- SWIM_CTR_* (11 words)
simCounters sim = allocaArray 11 $ \p -> c_simCounters sim p 11 >>= orFail sim >> peekArray 11 p

viewCapMax :: Int
viewCapMax = 256

getMembers :: Sim -> Word32 -> IO [CMember]                         -- members (Core.hs:76-77)
getMembers sim node = allocaArray viewCapMax $ \buf -> alloca $ \pn -> do
  c_getMembers sim node buf (fromIntegral viewCapMax) pn >>= orFail sim
  n <- peek pn
  peekArray (fromIntegral n) buf

setMembers :: Sim -> Word32 -> [CMember] -> IO ()                   -- swapTVar storeMembers (Spec.hs:101)
setMembers sim node ms = withArrayLen ms $ \n p -> c_setMembers sim node p (fromIntegral n) >>= orFail sim

kRandomMembers :: Sim -> Word32 -> Int -> [CMember] -> IO [CMember] -- Core.hs:69-74
kRandomMembers sim node n excludes =
  withArrayLen excludes $ \ne pe -> allocaArray viewCapMax $ \out -> alloca $ \pn -> do
    c_kRandom sim node (fromIntegral n) pe (fromIntegral ne) out (fromIntegral viewCapMax) pn >>= orFail sim
    k <- peek pn
    peekArray (fromIntegral k) out

removeDeadNodes :: Sim -> Word32 -> IO ()                           -- Core.hs:65-67
removeDeadNodes sim node = c_removeDead sim node >>= orFail sim

nextSeqNo, nextIncarnation :: Sim -> Word32 -> IO Int               -- Core.hs:49-53 (return the NEW value)
nextSeqNo sim node = alloca $ \p -> c_nextSeqNo sim node p >>= orFail sim >> fromIntegral <$> peek p
nextIncarnation sim node = alloca $ \p -> c_nextInc sim node p >>= orFail sim >> fromIntegral <$> peek p

applyWith :: (Sim -> Word32 -> Ptr CMessage -> Ptr CMessage -> Ptr CInt -> IO CInt)
          -> Sim -> Word32 -> CMessage -> IO (Maybe CMessage)
applyWith f sim node msg = with msg $ \pm -> alloca $ \po -> alloca $ \ph -> do
  f sim node pm po ph >>= orFail sim
  has <- peek ph
  if has /= 0 then Just <$> peek po else return Nothing

suspectNode, deadNode, aliveNode :: Sim -> Word32 -> CMessage -> IO (Maybe CMessage) -- Core.hs:189-218
suspectNode = applyWith c_suspectNode
deadNode    = applyWith c_deadNode
aliveNode   = applyWith c_aliveNode

handleMessage :: Sim -> Word32 -> (Word32, Word16) -> CMessage -> IO [CGossip]       -- process (Core.hs:89-117)
handleMessage sim node (addr, port) msg = with msg $ \pm -> allocaArray 2 $ \out -> alloca $ \pn -> do
  c_handleMessage sim node addr port pm out 2 pn >>= orFail sim
  n <- peek pn
  peekArray (fromIntegral n) out

broadcast :: Sim -> Word32 -> CMessage -> IO ()                     -- disseminate, Broadcast branch (Core.hs:131,136-138)
broadcast sim node msg = with msg $ \pm -> c_broadcast sim node pm >>= orFail sim

-- | SWIM_JOIN_FRESH: the joiners restart empty before they join.
joinFresh :: Word32
joinFresh = 1

-- | Join(joinHosts) for many processes at once, between steps: each (node, host) pair is one full-state exchange.
-- Returns (exchanges, inserted, full).
simJoin :: Sim -> Word32 -> [CJoin] -> IO (Word64, Word64, Word64)
simJoin sim flags js = withArrayLen js $ \n pj -> alloca $ \pe -> alloca $ \pn -> alloca $ \pf -> do
  c_simJoin sim pj (fromIntegral n) flags pe pn pf >>= orFail sim
  (,,) <$> peek pe <*> peek pn <*> peek pf

-- | memberlist's Leave for many processes at once, between steps: each listed process that is up goes down and its
-- members receive Dead about it, from it. Returns (left, delivered).
simLeave :: Sim -> [Word32] -> IO (Word64, Word64)
simLeave sim ids = withArrayLen ids $ \n pi' -> alloca $ \pl -> alloca $ \pd -> do
  c_simLeave sim pi' (fromIntegral n) pl pd >>= orFail sim
  (,) <$> peek pl <*> peek pd
